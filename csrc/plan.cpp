// plan.cpp — plan word stream -> typed trees -> device programs.
//
// Mirrors what the reference does at plan time, in this order:
//   ExecNode::create_tree / ExprNode::create_tree      src/exec/exec_node.cpp:347-394, src/expr/expr_node.cpp:401-445
//   ScalarFnCall::type_inferer                         src/expr/scalar_fn_call.cpp:40-120
//   FunctionManager::complete_fn                       src/expr/fn_manager.cpp:316-409
//   AggFnCall::type_inferer                            src/expr/agg_fn_call.cpp:87-122
//   Literal::get_value / cast_to_col_type              include/expr/literal.h:196-206
// and then lowers instead of interpreting: expressions become postfix bytecode whose operand
// classes are fixed here (no run-time type tags on the device).
#include "plan.h"
#include "hll.cuh"
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <functional>
#include <iterator>
#include <map>
#include "../include/bkgpu.h"
#include "datetime.h"
#include "in_set.h"

namespace bk {

constexpr int MAX_IN_LIST = 1 << 22;   // entries of one IN list (the planner writes an IN subquery's result rows into the plan as its list)
constexpr int MAX_IN_SETS = 256;       // IN sets of one plan (OP_IN_SET's b)

// ---------------------------------------------------------------- type helpers
static bool is_int_t(int t) { return t >= BK_INT8 && t <= BK_UINT64; }
static bool is_uint_t(int t) { return t >= BK_UINT8 && t <= BK_UINT64; }
static bool is_signed_t(int t) { return t >= BK_INT8 && t <= BK_INT64; }
static bool is_double_t(int t) { return t == BK_FLOAT || t == BK_DOUBLE; }
static bool is_datetime_family(int t) { return t == BK_DATETIME || t == BK_TIMESTAMP || t == BK_DATE || t == BK_TIME; }
static bool is_numeric_path_type(int t) { return t == BK_BOOL || is_int_t(t) || is_double_t(t) || is_datetime_family(t); }

int host_prim_class(int prim) {
    switch (prim) {
        case BK_FLOAT: case BK_DOUBLE: return VC_F64;
        case BK_BOOL: case BK_UINT8: case BK_UINT16: case BK_UINT32: case BK_UINT64:
        case BK_TIMESTAMP: case BK_DATE: case BK_DATETIME: return VC_U64;
        default: return VC_I64;
    }
}
int prim_storage(int prim) {  // src/common/common.cpp:514-544
    switch (prim) {
        case BK_INT8: case BK_INT16: case BK_INT32: case BK_TIME: return ST_I32;
        case BK_INT64: return ST_I64;
        case BK_UINT8: case BK_UINT16: case BK_UINT32: case BK_TIMESTAMP: case BK_DATE: return ST_U32;
        case BK_UINT64: case BK_DATETIME: return ST_U64;
        case BK_FLOAT: return ST_F32;
        case BK_DOUBLE: return ST_F64;
        case BK_BOOL: return ST_U8;
        case BK_STRING: return ST_BLOB16;
        case BK_HLL: return ST_HLL;
        default: return -1;
    }
}
int storage_bytes(int st) {
    switch (st) { case ST_I32: case ST_U32: case ST_F32: return 4; case ST_U8: return 1; case ST_BLOB16: return 16; case ST_HLL: return HLL_RAW_BYTES; default: return 8; }
}
static uint64_t dbits(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
static double bitsd(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }

// ExprValue::cast_to on canonical images, executed with the host's (x86-64) conversion semantics —
// the same ones the reference binary gets from its static_casts (expr_value.h:340-410,502-611).
uint64_t host_cast_prim(uint64_t v, int from, int to) {
    if (from != to && dt_is_family(from) && dt_is_family(to)) return dt_family_cast(v, from, to);   // (callers reject TIME sources first)
    int fc = host_prim_class(from);
    if (to == BK_DOUBLE || to == BK_FLOAT) {
        double d = fc == VC_F64 ? bitsd(v) : (fc == VC_U64 ? (double)v : (double)(int64_t)v);
        if (to == BK_FLOAT) d = (double)(float)d;
        return dbits(d);
    }
    if (to == BK_BOOL) return fc == VC_F64 ? (bitsd(v) != 0.0) : (v != 0);
    if (fc == VC_F64) {
        double d = bitsd(v);
        switch (to) {
            case BK_INT8: return (uint64_t)(int64_t)(int8_t)d;
            case BK_INT16: return (uint64_t)(int64_t)(int16_t)d;
            case BK_INT32: case BK_TIME: return (uint64_t)(int64_t)(int32_t)d;
            case BK_INT64: return (uint64_t)(int64_t)d;
            case BK_UINT8: return (uint64_t)(uint8_t)d;
            case BK_UINT16: return (uint64_t)(uint16_t)d;
            case BK_UINT32: case BK_TIMESTAMP: case BK_DATE: return (uint64_t)(uint32_t)d;
            default: return (uint64_t)d;
        }
    }
    switch (to) {
        case BK_INT8: return (uint64_t)(int64_t)(int8_t)v;
        case BK_INT16: return (uint64_t)(int64_t)(int16_t)v;
        case BK_INT32: case BK_TIME: return (uint64_t)(int64_t)(int32_t)v;
        case BK_UINT8: return (uint64_t)(uint8_t)v;
        case BK_UINT16: return (uint64_t)(uint16_t)v;
        case BK_UINT32: case BK_TIMESTAMP: case BK_DATE: return (uint64_t)(uint32_t)v;
        default: return v;
    }
}

// ---------------------------------------------------------------- reader
struct Reader {
    const int32_t* w; size_t n, pos = 0; bool fail = false; std::string err;
    int32_t rd() { if (pos >= n) { bad("truncated plan"); return 0; } return w[pos++]; }
    int64_t rd64() { uint32_t lo = (uint32_t)rd(), hi = (uint32_t)rd(); return (int64_t)(((uint64_t)hi << 32) | lo); }
    std::string rdstr() {
        int32_t len = rd();
        size_t words = ((size_t)(len < 0 ? 0 : len) + 3) / 4;
        if (len < 0 || len > 4096 || pos + words > n) { bad("bad string in plan"); return ""; }
        std::string s((const char*)(w + pos), (size_t)len); pos += words; return s;
    }
    void bad(const char* m) { if (!fail) { fail = true; err = m; } }
};

static bool is_literal_node(int nt) {
    return (nt >= BK_NULL_LITERAL && nt <= BK_STRING_LITERAL) || nt == BK_TIMESTAMP_LITERAL || nt == BK_DATETIME_LITERAL || nt == BK_DATE_LITERAL || nt == BK_TIME_LITERAL;
}

static void parse_enode(Reader& r, HExpr& e, int& remaining, int depth) {
    if (remaining <= 0 || depth > 64) { r.bad("expr node list does not match its node count"); return; }
    remaining--;
    e.node_type = r.rd(); e.col_type = r.rd();
    int nch = r.rd();
    switch (e.node_type) {
        case BK_SLOT_REF: e.tuple_id = r.rd(); e.slot_id = r.rd(); break;
        case BK_NULL_LITERAL: e.lit_null = true; e.lit_prim = BK_NULL_TYPE; break;
        case BK_BOOL_LITERAL: e.lit_bits = r.rd() ? 1 : 0; e.lit_prim = BK_BOOL; break;
        case BK_INT_LITERAL: e.lit_bits = (uint64_t)r.rd64(); e.lit_prim = BK_INT64; break;
        case BK_DOUBLE_LITERAL: e.lit_bits = (uint64_t)r.rd64(); e.lit_prim = BK_DOUBLE; break;
        case BK_STRING_LITERAL: e.lit_str = r.rdstr(); e.lit_prim = BK_STRING; break;   // (only where inference folds it into a date/time image)
        // DeriveExprNode.int_val carries the image (Literal::init, include/expr/literal.h:95-114)
        case BK_DATETIME_LITERAL: e.lit_bits = (uint64_t)r.rd64(); e.lit_prim = BK_DATETIME; break;
        case BK_TIMESTAMP_LITERAL: e.lit_bits = (uint64_t)(uint32_t)r.rd64(); e.lit_prim = BK_TIMESTAMP; break;
        case BK_DATE_LITERAL: e.lit_bits = (uint64_t)(uint32_t)r.rd64(); e.lit_prim = BK_DATE; break;
        case BK_TIME_LITERAL: e.lit_bits = (uint64_t)(int64_t)(int32_t)r.rd64(); e.lit_prim = BK_TIME; break;
        case BK_AGG_EXPR:
            e.name = r.rdstr(); e.tuple_id = r.rd(); e.final_slot = r.rd(); e.inter_slot = r.rd();
            // count_distinct / sum_distinct / avg_distinct are COUNT / SUM / AVG (name_type_map, agg_fn_call.cpp:32-40) that a MERGE_AGG node UPDATES
            // from its input rows instead of merging intermediates (AggFnCall::merge, agg_fn_call.cpp:719-727): the planner put the argument
            // into the GROUP BY of the aggregate below (select_planner.cpp:640-667), so each distinct value arrives once
            if (e.name == "count_distinct" || e.name == "sum_distinct" || e.name == "avg_distinct") { e.distinct = true; e.name.resize(e.name.size() - 9); }
            break;
        case BK_WINDOW_EXPR: e.name = r.rdstr(); e.tuple_id = r.rd(); e.slot_id = r.rd(); break;   // WindowFnCall::init (window_fn_call.cpp:19-63)
        case BK_FUNCTION_CALL: case BK_IS_NULL_PREDICATE: case BK_IN_PREDICATE: case BK_NOT_PREDICATE:
        case BK_AND_PREDICATE: case BK_OR_PREDICATE: case BK_XOR_PREDICATE: case BK_IS_TRUE_PREDICATE: {
            e.fn_op = r.rd(); e.name = r.rdstr();
            int na = r.rd();
            if (na < 0 || na > 8) { r.bad("bad n_arg_types"); return; }
            for (int i = 0; i < na; i++) e.arg_types.push_back(r.rd());
            e.return_type = r.rd();
        } break;
        case BK_LIKE_PREDICATE: case BK_ROW_EXPR:
            r.bad("LIKE / ROW expressions are outside the GPU path"); return;
        default: r.bad("unknown expr node type"); return;
    }
    if (e.node_type == BK_IN_PREDICATE && nch > MAX_IN_LIST + 1) {
        char buf[128];
        snprintf(buf, sizeof buf, "IN list of %d entries is longer than %d: outside the GPU path", nch - 1, MAX_IN_LIST);
        r.bad(buf); return;
    }
    if (nch < 0 || (nch > 1024 && e.node_type != BK_IN_PREDICATE)) { r.bad("bad expr num_children"); return; }
    // (a long list must be there before its children are allocated: each is a node of at least 3 words)
    if (nch > 1024 && (nch > remaining || (size_t)nch * 3 > r.n - r.pos)) { r.bad("expr node list does not match its node count"); return; }
    e.ch.resize((size_t)nch);
    for (int i = 0; i < nch && !r.fail; i++) parse_enode(r, e.ch[(size_t)i], remaining, depth + 1);
}
static void parse_expr(Reader& r, HExpr& e) {
    int n = r.rd();
    parse_enode(r, e, n, 0);
    if (!r.fail && n != 0) r.bad("expr node count mismatch");
}
static void parse_node(Reader& r, HNode& nd, int& remaining, int depth) {
    // (depth: a fragment has at most 64 nodes, so a chain of WINDOW -> SORT pairs — one per window function — nests that deep)
    if (remaining <= 0 || depth > 64) { r.bad("plan node list does not match its node count"); return; }
    remaining--;
    nd.node_type = r.rd();
    int nch = r.rd();
    nd.limit = r.rd64();
    auto exprs = [&](std::vector<HExpr>& v) {
        int n = r.rd();
        if (n < 0 || n > 256) { r.bad("bad expression count"); return; }
        v.resize((size_t)n);
        for (int i = 0; i < n && !r.fail; i++) parse_expr(r, v[(size_t)i]);
    };
    switch (nd.node_type) {
        case BK_SCAN_NODE: nd.tuple_id = r.rd(); (void)r.rd64(); break;
        case BK_WHERE_FILTER_NODE: case BK_TABLE_FILTER_NODE: case BK_HAVING_FILTER_NODE: exprs(nd.conjuncts); break;
        case BK_AGG_NODE: case BK_MERGE_AGG_NODE: nd.agg_tuple_id = r.rd(); exprs(nd.group_exprs); exprs(nd.agg_fns); break;
        case BK_SORT_NODE: {
            nd.tuple_id = r.rd();
            int n = r.rd();
            if (n < 0 || n > 64) { r.bad("bad order expr count"); return; }
            nd.order_exprs.resize((size_t)n);
            for (int i = 0; i < n && !r.fail; i++) {
                parse_expr(r, nd.order_exprs[(size_t)i]);
                nd.is_asc.push_back(r.rd()); nd.is_null_first.push_back(r.rd());
            }
        } break;
        case BK_JOIN_NODE: nd.join_type = r.rd(); exprs(nd.conjuncts); break;
        case BK_APPLY_NODE:
            nd.join_type = r.rd(); exprs(nd.conjuncts);
            nd.max_one_row = r.rd() != 0; nd.compare_type = r.rd(); nd.is_select_field = r.rd() != 0;
            break;
        case BK_LIMIT_NODE: nd.offset = r.rd64(); break;
        case BK_PACKET_NODE: case BK_SELECT_MANAGER_NODE: break;
        case BK_WINDOW_NODE: {   // pb::WindowNode: func_exprs, window_spec {partition_exprs, order_exprs, is_asc, window_frame}
            exprs(nd.agg_fns); exprs(nd.group_exprs);
            int n = r.rd();
            if (n < 0 || n > 64) { r.bad("bad order expr count"); return; }
            nd.order_exprs.resize((size_t)n);
            for (int i = 0; i < n && !r.fail; i++) { parse_expr(r, nd.order_exprs[(size_t)i]); nd.is_asc.push_back(r.rd()); }
            nd.has_frame = r.rd() != 0;
            if (nd.has_frame) {
                nd.frame_type = r.rd();
                for (HFrameBound* b : {&nd.frame_start, &nd.frame_end}) {
                    b->type = r.rd(); b->unbounded = r.rd() != 0; b->has_expr = r.rd() != 0;
                    if (b->has_expr && !r.fail) parse_expr(r, b->expr);
                }
            }
        } break;
        default: r.bad("plan node type outside the GPU path"); return;
    }
    if (nch < 0 || nch > 2) { r.bad("bad plan num_children"); return; }
    nd.ch.resize((size_t)nch);
    for (int i = 0; i < nch && !r.fail; i++) parse_node(r, nd.ch[(size_t)i], remaining, depth + 1);
}

// ---------------------------------------------------------------- type inference
struct Infer {
    const std::vector<HTuple>* tuples;
    std::string err;
    int code = 0;
    int slot_type(int tuple_id, int slot_id) const {
        for (auto& t : *tuples) if (t.tuple_id == tuple_id) for (auto& s : t.slots) if (s.first == slot_id) return s.second;
        return BK_INVALID_TYPE;
    }
    bool fail(int c, const char* fmt, ...) {
        char buf[256]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
        if (!code) { code = c; err = buf; }
        return false;
    }
};
static bool expr_constant(const HExpr& e) {
    if (e.node_type == BK_SLOT_REF || e.node_type == BK_AGG_EXPR) return false;
    for (auto& c : e.ch) if (!expr_constant(c)) return false;
    return true;
}
static void complete(HExpr& e, int nargs, int at, int rt) { e.arg_types.assign((size_t)nargs, at); e.return_type = rt; }

// named builtins of one / two DOUBLE arguments (src/expr/internal_functions.cpp:101-317,336-350) -> MathFn / Math2Fn, -1 = not one
static int math1_fn(const std::string& n) {
    static const std::pair<const char*, int> t[] = {{"sqrt", MF_SQRT}, {"sign", MF_SIGN}, {"sin", MF_SIN}, {"asin", MF_ASIN}, {"cos", MF_COS}, {"acos", MF_ACOS},
                                                    {"tan", MF_TAN}, {"cot", MF_COT}, {"atan", MF_ATAN}, {"ln", MF_LN}, {"bit_count", MF_BIT_COUNT}};
    for (auto& p : t) if (n == p.first) return p.second;
    return -1;
}
static int math2_fn(const std::string& n) {
    static const std::pair<const char*, int> t[] = {{"mod", MF2_FMOD}, {"log", MF2_LOG}, {"pow", MF2_POW}, {"power", MF2_POW}, {"greatest", MF2_GREATEST}, {"least", MF2_LEAST}};
    for (auto& p : t) if (n == p.first) return p.second;
    return -1;
}

// date-part and day-number functions (OP_DATEFN, datetime.h): name -> how the reference reads the argument and what it returns
// (internal_functions.cpp; return_type_map, fn_manager.cpp:184-243)
struct DateFnDef {
    const char* name;
    uint8_t fn;         // DateFn
    int arg_prim;       // the argument's cast_to before the computation (datediff: DATE, then TIMESTAMP)
    int ret;            // registered return type
    bool via_text;      // an INT64 argument is first written out as text (`if (in.type == pb::INT64) in.cast_to(pb::STRING)`)
    int extra;          // 0 = none, 1 = an optional mode after the value (week, yearweek), 2 = a unit before it (extract), 3 = a second value (datediff)
};
static const DateFnDef* date_fn_def(const std::string& n) {
    static const DateFnDef t[] = {
        {"year", DF_YEAR, BK_DATETIME, BK_UINT32, true, 0},            {"month", DF_MONTH, BK_DATETIME, BK_UINT32, true, 0},
        {"day", DF_DAY, BK_DATETIME, BK_UINT32, true, 0},              {"dayofmonth", DF_DAY, BK_DATETIME, BK_UINT32, true, 0},
        {"quarter", DF_QUARTER, BK_DATE, BK_INT32, false, 0},          {"hour", DF_HOUR, BK_TIME, BK_UINT32, false, 0},
        {"minute", DF_MINUTE, BK_TIME, BK_INT32, false, 0},            {"second", DF_SECOND, BK_TIME, BK_INT32, false, 0},
        {"dayofweek", DF_DAYOFWEEK, BK_DATETIME, BK_UINT32, true, 0},  {"weekday", DF_WEEKDAY, BK_DATETIME, BK_UINT32, true, 0},
        {"dayofyear", DF_DAYOFYEAR, BK_DATETIME, BK_UINT32, true, 0},  {"week", DF_WEEK, BK_DATETIME, BK_UINT32, false, 1},
        {"yearweek", DF_YEARWEEK, BK_DATETIME, BK_UINT32, false, 1},   {"weekofyear", DF_WEEKOFYEAR, BK_DATETIME, BK_UINT32, false, 0},
        {"to_days", DF_TO_DAYS, BK_TIMESTAMP, BK_INT64, false, 0},     {"to_seconds", DF_TO_SECONDS, BK_TIMESTAMP, BK_INT64, false, 0},
        {"unix_timestamp", DF_UNIX_TIMESTAMP, BK_TIMESTAMP, BK_INT64, true, 0},
        {"datediff", DF_DATEDIFF, BK_DATE, BK_INT32, true, 3},         {"extract", DF_EXTRACT, BK_TIMESTAMP, BK_UINT32, false, 2},
        {"date", DF_DATE, BK_DATETIME, BK_DATE, true, 0}};
    for (auto& d : t) if (n == d.name) return &d;
    return nullptr;
}
// date/time functions that stay on the CPU, and why
static const char* date_fn_refusal(const std::string& n) {
    static const std::pair<const char*, const char*> t[] = {
        {"date_add", "its registered return type differs from the type of the value it returns"}, {"date_sub", nullptr}, {"adddate", nullptr},
        {"subdate", nullptr}, {"timestampadd", nullptr}, {"timestampdiff", nullptr}, {"timediff", nullptr},
        {"now", "it reads the current time"}, {"sysdate", nullptr}, {"curdate", nullptr}, {"current_date", nullptr}, {"curtime", nullptr},
        {"current_time", nullptr}, {"current_timestamp", nullptr}, {"utc_timestamp", nullptr}, {"utc_date", nullptr}, {"utc_time", nullptr},
        {"date_format", "it returns STRING"}, {"dayname", nullptr}, {"monthname", nullptr}, {"time_format", nullptr},
        {"microsecond", "it is computed through the value's text"},
        {"time_to_sec", "its registered and run-time result types differ in sign"}, {"sec_to_time", nullptr},
        {"from_unixtime", "it is outside the GPU path"}, {"str_to_date", nullptr}, {"convert_tz", nullptr}};
    const char* why = nullptr;
    for (auto& p : t) {
        if (p.second) why = p.second;   // (an entry without a reason shares the one above it)
        if (n == p.first) return why;
    }
    return nullptr;
}

// A literal's value as the image of type `to` — ExprValue::cast_to (include/common/expr_value.h:502-611) on the host.
// `via_text`: Literal::cast_to_col_type (include/expr/literal.h:204-210) — a numeric literal that meets a date/time type is first
// written out in decimal and then read as a date ("20240131" -> 2024-01-31); a plain cast_to reinterprets the number as the image.
static bool fold_literal(Infer& in, HExpr& c, int to, bool via_text) {
    if (c.lit_null || to == BK_INVALID_TYPE || to == BK_NULL_TYPE) return true;
    if (c.lit_prim == BK_TIME && dt_is_family(to) && to != BK_TIME)
        return in.fail(BKGPU_EUNSUPPORTED, "a TIME value as DATE/DATETIME/TIMESTAMP depends on the current date: outside the GPU path");
    if (dt_is_family(to) && c.lit_prim != BK_STRING && !dt_is_family(c.lit_prim) && via_text) {
        if (is_double_t(c.lit_prim)) return in.fail(BKGPU_EUNSUPPORTED, "a DOUBLE literal compared as a date/time goes through its text form: outside the GPU path");
        char buf[32];
        if (is_uint_t(c.lit_prim)) snprintf(buf, sizeof buf, "%llu", (unsigned long long)c.lit_bits);
        else snprintf(buf, sizeof buf, "%lld", (long long)c.lit_bits);   // std::to_string, expr_value.h:709-726 (BOOL prints 0 / 1)
        c.lit_str = buf; c.lit_prim = BK_STRING;
    }
    if (c.lit_prim == BK_STRING) {
        if (to == BK_STRING) return true;
        if (!dt_is_family(to)) return in.fail(BKGPU_EUNSUPPORTED, "a STRING literal outside a date/time comparison is outside the GPU path");
        c.lit_bits = parse_literal(c.lit_str.c_str(), c.lit_str.size(), to);
    } else c.lit_bits = host_cast_prim(c.lit_bits, c.lit_prim, to);
    c.lit_prim = to;
    return true;
}

// A date function's arguments: date/time expressions are cast on the device, literals are folded here to the type the function
// casts them to; a non-literal number or string is refused (the reference would parse its text on every row).  extract's unit and
// week / yearweek's mode must be literals: they become the instruction's operand.
static bool infer_date_fn(Infer& in, HExpr& e, const DateFnDef& d) {
    const char* nm = e.name.c_str();
    const size_t n = e.ch.size(), v0 = d.extra == 2 ? 1 : 0, nv = d.extra == 3 ? 2 : 1;
    if (d.fn == DF_UNIX_TIMESTAMP && n == 0) return in.fail(BKGPU_EUNSUPPORTED, "unix_timestamp() without an argument reads the current time: outside the GPU path");
    if (d.extra == 1 ? (n < 1 || n > 2) : n != v0 + nv) return in.fail(BKGPU_EUNSUPPORTED, "%s() with %zu arguments is outside the GPU path", nm, n);
    for (size_t i = v0; i < v0 + nv; i++) {
        HExpr& c = e.ch[i];
        if (c.col_type == BK_TIME && d.arg_prim != BK_TIME)
            return in.fail(BKGPU_EUNSUPPORTED, "a TIME value as DATE/DATETIME/TIMESTAMP depends on the current date: outside the GPU path");
        if (is_literal_node(c.node_type)) {
            if (c.lit_null) continue;
            if (!fold_literal(in, c, d.arg_prim, d.via_text && c.lit_prim == BK_INT64)) return false;
            c.col_type = d.arg_prim;
        } else if (!dt_is_family(c.col_type))
            return in.fail(BKGPU_EUNSUPPORTED, "%s() over a non-literal argument of type %d: the reference parses its text on every row, outside the GPU path", nm, c.col_type);
    }
    if (d.extra == 1 && n == 2) {
        const HExpr& m = e.ch[1];
        if (!is_literal_node(m.node_type) || m.lit_null || !(is_int_t(m.lit_prim) || m.lit_prim == BK_BOOL))
            return in.fail(BKGPU_EUNSUPPORTED, "%s() takes a literal integer mode", nm);
    }
    if (d.extra == 2 && !is_literal_node(e.ch[0].node_type)) return in.fail(BKGPU_EUNSUPPORTED, "extract() takes a literal unit");
    e.arg_types.clear();   // named builtins cast nothing on the way in (complete_common_fn)
    e.return_type = d.ret;
    if (!e.col_type) e.col_type = d.ret;
    return true;
}

static bool infer_expr(Infer& in, HExpr& e) {
    for (auto& c : e.ch) if (!infer_expr(in, c)) return false;
    e.is_constant = expr_constant(e);
    auto all_int = [&](const std::vector<int>& t) { for (int x : t) if (!is_int_t(x)) return false; return true; };
    auto has = [&](const std::vector<int>& t, bool (*f)(int)) { for (int x : t) if (f(x)) return true; return false; };
    auto has_eq = [&](const std::vector<int>& t, int v) { for (int x : t) if (x == v) return true; return false; };
    switch (e.node_type) {
        case BK_SLOT_REF: {
            int st = in.slot_type(e.tuple_id, e.slot_id);
            if (e.col_type == BK_INVALID_TYPE) e.col_type = st;
            if (e.col_type == BK_INVALID_TYPE) return in.fail(BKGPU_EINVAL, "slot %d_%d has no tuple descriptor", e.tuple_id, e.slot_id);
            if (!is_numeric_path_type(e.col_type) && e.col_type != BK_STRING)
                return in.fail(BKGPU_EUNSUPPORTED, "column %d_%d has type %d, outside the GPU path", e.tuple_id, e.slot_id, e.col_type);
            return true;
        }
        case BK_NULL_LITERAL: if (!e.col_type) e.col_type = BK_NULL_TYPE; return true;
        case BK_BOOL_LITERAL: if (!e.col_type) e.col_type = BK_BOOL; return true;
        case BK_INT_LITERAL: if (!e.col_type) e.col_type = BK_INT64; return true;
        case BK_DOUBLE_LITERAL: if (!e.col_type) e.col_type = BK_DOUBLE; return true;
        case BK_STRING_LITERAL: if (!e.col_type) e.col_type = BK_STRING; return true;
        case BK_DATETIME_LITERAL: if (!e.col_type) e.col_type = BK_DATETIME; return true;
        case BK_TIMESTAMP_LITERAL: if (!e.col_type) e.col_type = BK_TIMESTAMP; return true;
        case BK_DATE_LITERAL: if (!e.col_type) e.col_type = BK_DATE; return true;
        case BK_TIME_LITERAL: if (!e.col_type) e.col_type = BK_TIME; return true;
        case BK_AGG_EXPR: {  // agg_fn_call.cpp:87-122
            int ct = e.ch.empty() ? BK_INVALID_TYPE : e.ch[0].col_type;
            if (e.name == "count_star" || e.name == "count") e.col_type = BK_INT64;
            else if (e.name == "avg") e.col_type = BK_DOUBLE;
            else if (e.name == "sum") {
                if (e.ch.empty()) return in.fail(BKGPU_EINVAL, "sum() without an argument");
                e.col_type = is_double_t(ct) ? BK_DOUBLE : (is_uint_t(ct) ? BK_UINT64 : BK_INT64);
            } else if (e.name == "min" || e.name == "max") {
                if (e.ch.empty()) return in.fail(BKGPU_EINVAL, "%s() without an argument", e.name.c_str());
                e.col_type = ct;
            } else if (e.name == "hll_add_agg") {   // agg_fn_call.cpp:124-130
                if (e.ch.empty()) return in.fail(BKGPU_EINVAL, "hll_add_agg() without an argument");
                if (ct == BK_STRING)
                    return in.fail(BKGPU_EUNSUPPORTED, "hll_add_agg over a STRING argument is outside the GPU path: a dictionary code would be hashed, not the text");
                if (ct != BK_NULL_TYPE && !hll_key_bytes(ct)) return in.fail(BKGPU_EUNSUPPORTED, "hll_add_agg over an argument of type %d is outside the GPU path", ct);
                e.col_type = BK_HLL;
            } else if (e.name == "rb_build_agg") {   // agg_fn_call.cpp:132-141: BITMAP; update adds get_numberic<uint32_t>(value) (:642-651)
                if (e.ch.empty()) return in.fail(BKGPU_EINVAL, "rb_build_agg() without an argument");
                if (is_double_t(ct))
                    return in.fail(BKGPU_EUNSUPPORTED, "rb_build_agg over a FLOAT / DOUBLE argument is outside the GPU path: only integer and BOOL values are lowered");
                if (ct == BK_STRING)
                    return in.fail(BKGPU_EUNSUPPORTED, "rb_build_agg over a STRING argument is outside the GPU path: a dictionary code would be added, not the value");
                if (ct == BK_DATETIME || ct == BK_TIMESTAMP || ct == BK_DATE || ct == BK_TIME)
                    return in.fail(BKGPU_EUNSUPPORTED, "rb_build_agg over a date / time argument (type %d) is outside the GPU path", ct);
                if (ct != BK_NULL_TYPE && ct != BK_BOOL && !is_int_t(ct)) return in.fail(BKGPU_EUNSUPPORTED, "rb_build_agg over an argument of type %d is outside the GPU path", ct);
                e.col_type = BK_BITMAP;
            } else if (e.name == "hll_merge_agg") {
                return in.fail(BKGPU_EUNSUPPORTED, "hll_merge_agg over stored sketches is outside the GPU path: a DENSE or SPARSE sketch varies in length");
            } else return in.fail(BKGPU_EUNSUPPORTED, "aggregate '%s' is outside the GPU path", e.name.c_str());
            if (e.name != "count_star" && e.name != "count" && !e.ch.empty() && ct == BK_STRING)
                return in.fail(BKGPU_EUNSUPPORTED, "%s over a STRING argument is outside the GPU path", e.name.c_str());
            return true;
        }
        case BK_WINDOW_EXPR: {   // WindowFnCall::type_inferer (window_fn_call.cpp:206-285)
            const int ct = e.ch.empty() ? BK_INVALID_TYPE : e.ch[0].col_type;
            const std::string& n = e.name;
            if (n == "count_star" || n == "count" || n == "row_number" || n == "rank" || n == "dense_rank" || n == "ntile") e.col_type = BK_INT64;
            else if (n == "avg" || n == "percent_rank" || n == "cume_dist") e.col_type = BK_DOUBLE;
            else if (n == "sum") {
                if (e.ch.empty()) return in.fail(BKGPU_EINVAL, "window sum() without an argument");
                e.col_type = is_double_t(ct) || ct == BK_STRING ? BK_DOUBLE : BK_INT64;
            } else if (n == "min" || n == "max" || n == "lead" || n == "lag" || n == "first_value" || n == "last_value" || n == "nth_value") {
                if (e.ch.empty()) return in.fail(BKGPU_EINVAL, "window %s() without an argument", n.c_str());
                e.col_type = ct;
            } else return in.fail(BKGPU_EUNSUPPORTED, "window function '%s' is outside the GPU path", n.c_str());
            return true;
        }
        case BK_AND_PREDICATE: case BK_OR_PREDICATE: case BK_XOR_PREDICATE: case BK_NOT_PREDICATE:
        case BK_IS_NULL_PREDICATE: case BK_IS_TRUE_PREDICATE:
            if (!e.col_type) e.col_type = BK_BOOL;
            return true;
        case BK_IN_PREDICATE: {  // InPredicate::singel_open, predicate.cpp:102-148
            if (e.ch.size() < 2) return in.fail(BKGPU_EINVAL, "IN without a value list");
            if (e.ch[0].node_type == BK_SLOT_REF)
                for (size_t i = 1; i < e.ch.size(); i++) if (e.ch[i].is_constant) e.ch[i].col_type = e.ch[0].col_type;
            std::vector<int> types = {e.ch[0].col_type, e.ch[1].col_type};
            int map_type;
            if (all_int(types)) map_type = BK_INT64;
            else if (has_eq(types, BK_DATETIME)) map_type = BK_DATETIME;     // InPredicate::singel_open, predicate.cpp:102-119
            else if (has_eq(types, BK_TIMESTAMP)) map_type = BK_TIMESTAMP;
            else if (has_eq(types, BK_DATE)) map_type = BK_DATE;
            else if (has_eq(types, BK_TIME)) map_type = BK_TIME;
            else if (has(types, is_double_t) || has(types, is_int_t)) map_type = BK_DOUBLE;
            else return in.fail(BKGPU_EUNSUPPORTED, "IN over STRING is outside the GPU path");
            if (e.ch[0].col_type == BK_STRING) return in.fail(BKGPU_EUNSUPPORTED, "IN over a STRING operand is outside the GPU path");
            if (e.ch[0].col_type == BK_TIME && map_type != BK_TIME && dt_is_family(map_type))
                return in.fail(BKGPU_EUNSUPPORTED, "a TIME value as DATE/DATETIME/TIMESTAMP depends on the current date: outside the GPU path");
            for (size_t i = 1; i < e.ch.size(); i++) {
                HExpr& c = e.ch[i];
                if (!is_literal_node(c.node_type)) return in.fail(BKGPU_EUNSUPPORTED, "IN list entries must be literals");
                // Literal::get_value casts to the literal's col_type, then the set takes value.cast_to(_map_type) (predicate.cpp:120-136)
                if (!fold_literal(in, c, c.col_type, false) || !fold_literal(in, c, map_type, false)) return false;
                if (!c.lit_null) c.col_type = map_type;
            }
            e.arg_types.assign(1, map_type);
            if (!e.col_type) e.col_type = BK_BOOL;
            return true;
        }
        default: break;
    }
    // FUNCTION_CALL
    if (e.fn_op == BK_FT_COMMON) {
        if (const DateFnDef* d = date_fn_def(e.name)) return infer_date_fn(in, e, *d);
        if (const char* why = date_fn_refusal(e.name)) return in.fail(BKGPU_EUNSUPPORTED, "%s() is outside the GPU path: %s", e.name.c_str(), why);
    }
    if (!e.arg_types.empty() && e.return_type != BK_INVALID_TYPE) {  // completed by the db already
        if (!e.col_type) e.col_type = e.return_type;
    } else {
        switch (e.fn_op) {  // predicates take the column's type: scalar_fn_call.cpp:57-67
            case BK_FT_EQ: case BK_FT_NE: case BK_FT_GE: case BK_FT_GT: case BK_FT_LE: case BK_FT_LT:
                if (e.ch.size() == 2 && e.ch[0].node_type == BK_SLOT_REF && e.ch[1].is_constant) e.ch[1].col_type = e.ch[0].col_type;
                break;
            default: break;
        }
        std::vector<int> types;
        for (auto& c : e.ch) {
            if (c.col_type == BK_INVALID_TYPE) return in.fail(BKGPU_EINVAL, "child of fn_op %d has INVALID_TYPE", e.fn_op);
            types.push_back(c.col_type);
        }
        switch (e.fn_op) {  // fn_manager.cpp:316-409
            case BK_FT_EQ: case BK_FT_NE: case BK_FT_GE: case BK_FT_GT: case BK_FT_LE: case BK_FT_LT:
                if (types.size() != 2) return in.fail(BKGPU_EINVAL, "comparison needs two operands");
                if (all_int(types)) complete(e, 2, has(types, is_uint_t) ? BK_UINT64 : BK_INT64, BK_BOOL);
                else if (has_eq(types, BK_DATETIME)) complete(e, 2, BK_DATETIME, BK_BOOL);
                else if (has_eq(types, BK_TIMESTAMP)) complete(e, 2, BK_TIMESTAMP, BK_BOOL);
                else if (has_eq(types, BK_DATE)) complete(e, 2, BK_DATE, BK_BOOL);
                else if (has_eq(types, BK_TIME)) complete(e, 2, BK_TIME, BK_BOOL);
                else if (has(types, is_double_t)) complete(e, 2, BK_DOUBLE, BK_BOOL);
                else if (has(types, is_int_t)) complete(e, 2, BK_DOUBLE, BK_BOOL);
                else complete(e, 2, BK_STRING, BK_BOOL);
                break;
            case BK_FT_ADD: case BK_FT_MINUS: case BK_FT_MULTIPLIES:
                if (types.size() != 2) return in.fail(BKGPU_EINVAL, "arithmetic needs two operands");
                if (has(types, is_double_t)) complete(e, 2, BK_DOUBLE, BK_DOUBLE);
                else if (has(types, is_uint_t)) complete(e, 2, BK_UINT64, BK_UINT64);
                else complete(e, 2, BK_INT64, BK_INT64);
                break;
            case BK_FT_DIVIDES: complete(e, 2, BK_DOUBLE, BK_DOUBLE); break;
            case BK_FT_MOD:
                if (has(types, is_uint_t)) complete(e, 2, BK_UINT64, BK_UINT64); else complete(e, 2, BK_INT64, BK_INT64);
                break;
            case BK_FT_BIT_AND: case BK_FT_BIT_OR: case BK_FT_BIT_XOR: case BK_FT_LS: case BK_FT_RS:
                complete(e, 2, BK_UINT64, BK_UINT64); break;
            case BK_FT_BIT_NOT: complete(e, 1, BK_UINT64, BK_UINT64); break;
            case BK_FT_UMINUS:
                if (has(types, is_double_t)) complete(e, 1, BK_DOUBLE, BK_DOUBLE);
                else if (has(types, is_uint_t)) complete(e, 1, BK_UINT64, BK_UINT64);
                else complete(e, 1, BK_INT64, BK_INT64);
                break;
            case BK_FT_LOGIC_NOT: complete(e, 1, BK_BOOL, BK_BOOL); break;
            case BK_FT_COMMON: {   // return_type_map + complete_common_fn (fn_manager.cpp:398-401,466-514); no argument casts
                std::vector<int> merge;
                const size_t n = types.size();
                if (e.name == "if") { if (n != 3) return in.fail(BKGPU_EINVAL, "if() needs three arguments"); merge = {types[1], types[2]}; }
                else if (e.name == "ifnull") { if (n != 2) return in.fail(BKGPU_EINVAL, "ifnull() needs two arguments"); merge = {types[0], types[1]}; }
                else if (e.name == "case_when") {
                    if (n < 2) return in.fail(BKGPU_EINVAL, "case_when needs a WHEN/THEN pair");
                    for (size_t i = 1; i < n; i++) if (i % 2 == 1 || i + 1 == n) merge.push_back(types[i]);
                }
                else if (e.name == "abs" || e.name == "round" || e.name == "cast_to_double" || math1_fn(e.name) >= 0 || math2_fn(e.name) >= 0 || e.name == "pi") e.return_type = BK_DOUBLE;
                else if (e.name == "floor" || e.name == "ceil" || e.name == "ceiling" || e.name == "cast_to_signed") e.return_type = BK_INT64;
                else if (e.name == "cast_to_unsigned") e.return_type = BK_UINT64;
                else return in.fail(BKGPU_EUNSUPPORTED, "function '%s' is outside the GPU path", e.name.c_str());
                if (!merge.empty()) {   // has_merged_type (include/common/type_utils.h:502-560)
                    bool all_null = true, all_equal = true, all_num = true, has_dbl = false, has_u64 = false, has_signed = false;
                    int first = BK_NULL_TYPE;
                    for (int t : merge) {
                        if (t == BK_NULL_TYPE) continue;
                        if (all_null) { first = t; all_null = false; }
                        if (t != first) all_equal = false;
                        if (!(is_double_t(t) || is_int_t(t) || t == BK_BOOL)) all_num = false;
                        if (is_double_t(t)) has_dbl = true;
                        if (t == BK_UINT64) has_u64 = true;
                        if (t == BK_INT8 || t == BK_INT16 || t == BK_INT32 || t == BK_INT64) has_signed = true;
                    }
                    if (all_null) return in.fail(BKGPU_EUNSUPPORTED, "%s: every branch is NULL", e.name.c_str());
                    if (all_equal) e.return_type = first;
                    else if (all_num) e.return_type = has_dbl ? BK_DOUBLE : (has_u64 ? (has_signed ? BK_DOUBLE : BK_UINT64) : BK_INT64);
                    else return in.fail(BKGPU_EUNSUPPORTED, "%s over date/time or STRING branches is outside the GPU path", e.name.c_str());
                    if (e.return_type == BK_STRING || is_datetime_family(e.return_type))
                        return in.fail(BKGPU_EUNSUPPORTED, "%s returning type %d is outside the GPU path", e.name.c_str(), e.return_type);
                }
                if (e.name == "sign" || e.name == "bit_count") e.return_type = BK_INT64;   // return_type_map, fn_manager.cpp:105-128
                if ((e.name == "abs" || e.name == "floor" || e.name == "ceil" || e.name == "ceiling" || e.name.rfind("cast_to_", 0) == 0 || math1_fn(e.name) >= 0) && n != 1)
                    return in.fail(BKGPU_EINVAL, "%s() needs one argument", e.name.c_str());
                if (e.name == "pi" && n != 0) return in.fail(BKGPU_EINVAL, "pi() takes no argument");
                if (math2_fn(e.name) >= 0 && (e.name == "greatest" || e.name == "least" ? n < 1 : n != 2))
                    return in.fail(BKGPU_EINVAL, "%s() needs %s", e.name.c_str(), e.name == "greatest" || e.name == "least" ? "an argument" : "two arguments");
                if (e.name == "round" && (n < 1 || n > 2 || (n == 2 && (!is_literal_node(e.ch[1].node_type) || e.ch[1].lit_null))))
                    return in.fail(BKGPU_EUNSUPPORTED, "round() needs a literal number of decimals");
                for (auto& c : e.ch)
                    if (c.col_type == BK_STRING || is_datetime_family(c.col_type)) return in.fail(BKGPU_EUNSUPPORTED, "%s over STRING / date-time arguments", e.name.c_str());
            } break;
            default: return in.fail(BKGPU_EUNSUPPORTED, "function fn_op=%d name='%s' is outside the GPU path", e.fn_op, e.name.c_str());
        }
        if (!e.col_type) e.col_type = e.return_type;
        // Literal::cast_to_col_type on literal children (scalar_fn_call.cpp:113-117)
        for (size_t i = 0; i < e.arg_types.size() && i < e.ch.size(); i++) {
            HExpr& c = e.ch[i];
            if (is_literal_node(c.node_type) && !c.lit_null) {
                if (!fold_literal(in, c, e.arg_types[i], true)) return false;
                c.col_type = e.arg_types[i];   // value_to_node_type: the literal now is of the argument's type (literal.h:296-310)
            }
        }
    }
    if (e.ch.size() < e.arg_types.size()) return in.fail(BKGPU_EINVAL, "function has fewer children than arg_types");
    for (int at : e.arg_types)
        if (at == BK_STRING) return in.fail(BKGPU_EUNSUPPORTED, "STRING-domain comparison is outside the GPU path");
    for (size_t i = 0; i < e.arg_types.size(); i++) {
        if (e.ch[i].col_type == BK_TIME && e.arg_types[i] != BK_TIME && dt_is_family(e.arg_types[i]))
            return in.fail(BKGPU_EUNSUPPORTED, "a TIME value as DATE/DATETIME/TIMESTAMP depends on the current date: outside the GPU path");
        if (e.ch[i].col_type == BK_STRING) return in.fail(BKGPU_EUNSUPPORTED, "STRING operands are outside the GPU path");
    }
    return true;
}

// ---------------------------------------------------------------- lowering
static bool is_filter(const HNode* n) {
    return n && (n->node_type == BK_WHERE_FILTER_NODE || n->node_type == BK_TABLE_FILTER_NODE);
}

// FilterNode passes a row when every conjunct is non-NULL true (filter_node.cpp:726-734); one OP_AND takes at most 8 of them
static bool at_most_8_conjuncts(Infer& in, size_t n, const std::string& where) {
    return n <= 8 || in.fail(BKGPU_EUNSUPPORTED, "more than 8 conjuncts%s", where.c_str());
}

// lowers expressions into one program; its constants are numbered from 0
struct Lower {
    Compiled* out;
    Infer* in;
    Program* p;
    int n_const = 0;
    int intern_col(int tuple_id, int slot_id, int prim) {
        auto& cols = out->cols;
        for (size_t i = 0; i < cols.size(); i++) if (cols[i].tuple_id == tuple_id && cols[i].slot_id == slot_id) return (int)i;
        cols.push_back({tuple_id, slot_id, prim});
        out->col_side.push_back(out->build_tuple >= 0 && tuple_id == out->build_tuple ? 1 : 0);
        return (int)cols.size() - 1;
    }
    bool emit(uint8_t op, uint8_t a = 0, uint8_t b = 0, uint8_t c = 0) {
        if (p->n_instr >= MAX_INSTR) return in->fail(BKGPU_EUNSUPPORTED, "expression too long for the device program (%d instructions)", MAX_INSTR);
        p->code[p->n_instr++] = Instr{op, a, b, c};
        return true;
    }
    int add_const(uint64_t bits, bool isnull) {
        if (n_const >= MAX_CONST) { in->fail(BKGPU_EUNSUPPORTED, "too many constants (%d)", MAX_CONST); return -1; }
        int i = n_const++;
        p->cbits[i] = bits;
        if (isnull) p->cnull |= 1ull << i;
        return i;
    }
    // ExprValue::cast_to between canonical images: a no-op when the image does not change
    bool cast(int from, int to) {
        if (from == to || to == BK_INVALID_TYPE || from == BK_NULL_TYPE) return true;
        if (dt_is_family(from) && dt_is_family(to)) return emit(OP_CAST, (uint8_t)from, (uint8_t)to);   // calendar conversion (datetime.h)
        bool from_int = is_int_t(from) || from == BK_BOOL || is_datetime_family(from);
        if (from_int && (to == BK_INT64 || to == BK_UINT64 || to == BK_DATETIME)) return true;  // sign/zero-extended image reinterpreted
        if (from == BK_FLOAT && to == BK_DOUBLE) return true;                                    // floats travel widened
        return emit(OP_CAST, (uint8_t)from, (uint8_t)to);
    }
    // emits code leaving the value on the stack; returns false on error.  `stack` tracks depth.
    bool expr(const HExpr& e, int& depth) {
        if (depth + 1 > STACK_DEPTH - 1) return in->fail(BKGPU_EUNSUPPORTED, "expression nests deeper than the device stack");
        switch (e.node_type) {
            case BK_SLOT_REF: {
                int st = in->slot_type(e.tuple_id, e.slot_id);
                if (st == BK_INVALID_TYPE) st = e.col_type;
                if (st == BK_STRING) return in->fail(BKGPU_EUNSUPPORTED, "STRING column %d_%d used in an expression", e.tuple_id, e.slot_id);
                int ci = intern_col(e.tuple_id, e.slot_id, st);
                if (ci >= MAX_COLS) return in->fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
                if (!emit(OP_LOAD_COL, (uint8_t)ci, 0, (uint8_t)out->col_side[(size_t)ci])) return false;  // c = 1: read at the matched build row
                depth++;
                return cast(st, e.col_type);
            }
            case BK_NULL_LITERAL: { int k = add_const(0, true); if (k < 0) return false; depth++; return emit(OP_CONST, (uint8_t)k); }
            case BK_BOOL_LITERAL: case BK_INT_LITERAL: case BK_DOUBLE_LITERAL: case BK_STRING_LITERAL:
            case BK_DATETIME_LITERAL: case BK_TIMESTAMP_LITERAL: case BK_DATE_LITERAL: case BK_TIME_LITERAL: {
                if (e.lit_prim == BK_STRING) return in->fail(BKGPU_EUNSUPPORTED, "a STRING literal outside a date/time comparison is outside the GPU path");
                if (e.lit_prim == BK_TIME && e.col_type != BK_TIME && dt_is_family(e.col_type))
                    return in->fail(BKGPU_EUNSUPPORTED, "a TIME value as DATE/DATETIME/TIMESTAMP depends on the current date: outside the GPU path");
                // Literal::get_value: _value.cast_to(_col_type)
                uint64_t bits = e.col_type ? host_cast_prim(e.lit_bits, e.lit_prim, e.col_type) : e.lit_bits;
                int k = add_const(bits, false); if (k < 0) return false;
                depth++;
                return emit(OP_CONST, (uint8_t)k);
            }
            case BK_AND_PREDICATE: case BK_OR_PREDICATE: {
                if (e.ch.empty() || e.ch.size() > 8) return in->fail(BKGPU_EUNSUPPORTED, "AND/OR with %zu operands", e.ch.size());
                int d0 = depth;
                for (auto& c : e.ch) { if (!expr(c, depth)) return false; if (!to_bool(c)) return false; }
                depth = d0 + 1;
                return emit(e.node_type == BK_AND_PREDICATE ? OP_AND : OP_OR, (uint8_t)e.ch.size());
            }
            case BK_XOR_PREDICATE: {
                if (e.ch.size() != 2) return in->fail(BKGPU_EINVAL, "XOR needs two operands");
                for (auto& c : e.ch) { if (!expr(c, depth)) return false; if (!to_bool(c)) return false; }
                depth--;
                return emit(OP_XOR);
            }
            case BK_NOT_PREDICATE: case BK_IS_TRUE_PREDICATE: {
                if (e.ch.size() != 1) return in->fail(BKGPU_EINVAL, "unary predicate needs one operand");
                if (!expr(e.ch[0], depth) || !to_bool(e.ch[0])) return false;
                return emit(e.node_type == BK_NOT_PREDICATE ? OP_NOT3 : OP_IS_TRUE);
            }
            case BK_IS_NULL_PREDICATE:
                if (e.ch.size() != 1) return in->fail(BKGPU_EINVAL, "IS NULL needs one operand");
                if (!expr(e.ch[0], depth)) return false;
                return emit(OP_IS_NULL);
            case BK_IN_PREDICATE: {
                int map_type = e.arg_types[0];
                if (!expr(e.ch[0], depth) || !cast(e.ch[0].col_type, map_type)) return false;
                int first = n_const, cnt = 0; bool has_null = false;
                for (size_t i = 1; i < e.ch.size(); i++) { if (e.ch[i].lit_null) has_null = true; else cnt++; }
                const uint8_t flags = (uint8_t)((has_null ? 16 : 0) | host_prim_class(map_type));
                if (cnt > 255 || n_const + cnt > MAX_CONST) {   // a list the constant pool cannot hold is probed as a hashed set
                    const int s = in_set(e, map_type, has_null), k = s < 0 ? -1 : add_const(0, false);
                    return k >= 0 && emit(OP_IN_SET, (uint8_t)k, (uint8_t)s, flags);
                }
                for (size_t i = 1; i < e.ch.size(); i++)
                    if (!e.ch[i].lit_null && add_const(in_entry(e.ch[i], map_type), false) < 0) return false;
                return emit(OP_IN, (uint8_t)first, (uint8_t)cnt, flags);
            }
            case BK_FUNCTION_CALL: {
                if (e.fn_op == BK_FT_COMMON) return common_fn(e, depth);
                int d0 = depth;
                for (size_t i = 0; i < e.ch.size(); i++) {
                    if (!expr(e.ch[i], depth)) return false;
                    if (i < e.arg_types.size() && !cast(e.ch[i].col_type, e.arg_types[i])) return false;
                }
                int at = e.arg_types.empty() ? BK_INT64 : e.arg_types[0];
                uint8_t vc = (uint8_t)host_prim_class(at);
                bool ok;
                switch (e.fn_op) {
                    case BK_FT_EQ: case BK_FT_NE: case BK_FT_GT: case BK_FT_GE: case BK_FT_LT: case BK_FT_LE:
                        ok = emit(OP_CMP, (uint8_t)e.fn_op, vc); depth = d0 + 1; break;
                    case BK_FT_ADD: case BK_FT_MINUS: case BK_FT_MULTIPLIES: ok = emit(OP_ARITH, (uint8_t)e.fn_op, vc); depth = d0 + 1; break;
                    case BK_FT_DIVIDES: ok = emit(OP_DIV_F64); depth = d0 + 1; break;
                    case BK_FT_MOD: ok = emit(OP_MOD, 0, vc); depth = d0 + 1; break;
                    case BK_FT_BIT_AND: case BK_FT_BIT_OR: case BK_FT_BIT_XOR: case BK_FT_LS: case BK_FT_RS:
                        ok = emit(OP_BIT, (uint8_t)e.fn_op); depth = d0 + 1; break;
                    case BK_FT_BIT_NOT: ok = emit(OP_BIT_NOT); break;
                    case BK_FT_UMINUS: ok = emit(OP_NEG, 0, vc); break;   // minus_uint yields the INT64 image too (operators.cpp:31)
                    case BK_FT_LOGIC_NOT: ok = emit(OP_LOGIC_NOT); break;
                    default: return in->fail(BKGPU_EUNSUPPORTED, "fn_op %d", e.fn_op);
                }
                if (!ok) return false;
                int rt = e.return_type;
                if (e.fn_op == BK_FT_UMINUS && at == BK_UINT64) rt = BK_INT64;
                return cast(rt, e.col_type);  // _fn_call(args).cast_to(_col_type)
            }
            default: return in->fail(BKGPU_EUNSUPPORTED, "expr node type %d cannot be lowered", e.node_type);
        }
    }
    // an IN list entry as the image of the set's type
    static uint64_t in_entry(const HExpr& c, int map_type) {
        const uint64_t bits = c.col_type ? host_cast_prim(c.lit_bits, c.lit_prim, c.col_type) : c.lit_bits;   // Literal::get_value
        return host_cast_prim(bits, c.col_type ? c.col_type : c.lit_prim, map_type);                          // value.cast_to(_map_type)
    }
    // the set of `e`'s entries: built at its first lowering, found again at the next (jfast lowers the same expressions)
    int in_set(const HExpr& e, int map_type, bool has_null) {
        InSets& reg = *out->in_sets;
        for (auto& x : reg.of_expr) if (x.first == &e) return x.second;
        if ((int)reg.sets.size() >= MAX_IN_SETS) { in->fail(BKGPU_EUNSUPPORTED, "more than %d long IN lists in one plan", MAX_IN_SETS); return -1; }
        std::vector<uint64_t> v;
        v.reserve(e.ch.size() - 1);
        for (size_t i = 1; i < e.ch.size(); i++) if (!e.ch[i].lit_null) v.push_back(in_entry(e.ch[i], map_type));
        InSet s;
        s.vclass = host_prim_class(map_type);
        s.has_null = has_null;
        s.image = in_set_build(v.data(), v.size(), s.vclass, &s.n_distinct);
        reg.sets.push_back(std::move(s));
        reg.of_expr.push_back({&e, (int)reg.sets.size() - 1});
        return (int)reg.sets.size() - 1;
    }
    // named builtins (FT_COMMON): arguments are NOT cast (arg_types stay empty), the result is cast to the node's col_type
    bool branch(const HExpr& c, int to, int& depth) { return expr(c, depth) && cast(c.col_type, to); }
    // a date function: the argument, its cast_to (OP_CAST), then OP_DATEFN; a call over literals alone is computed here instead
    bool date_fn(const HExpr& e, const DateFnDef& d, int& depth) {
        const int d0 = depth;
        const size_t v0 = d.extra == 2 ? 1 : 0, nv = d.extra == 3 ? 2 : 1;
        int arg = 0;
        bool is_null = false;   // an unknown extract unit or a NULL literal argument: the call is NULL
        if (d.extra == 1) arg = e.ch.size() == 2 ? (int)((uint32_t)e.ch[1].lit_bits % 8) : DT_NO_MODE;   // get_numberic<uint32_t>() % 8
        if (d.extra == 2) {                                                                                  // input[0].str_val == "year" ...
            static const char* const units[] = {"year", "month", "day", "hour", "minute", "second"};
            const HExpr& u = e.ch[0];
            arg = -1;
            for (int i = 0; i < 6; i++) if (!u.lit_null && u.lit_prim == BK_STRING && u.lit_str == units[i]) arg = i;
            is_null = arg < 0;
        }
        bool all_literal = true;
        uint64_t img[2] = {0, 0};
        for (size_t i = 0; i < nv; i++) {
            const HExpr& c = e.ch[v0 + i];
            if (!is_literal_node(c.node_type)) { all_literal = false; continue; }
            if (c.lit_null) is_null = true;
            else img[i] = d.fn == DF_DATEDIFF ? host_cast_prim(c.lit_bits, BK_DATE, BK_TIMESTAMP) : c.lit_bits;   // (already the argument's type)
        }
        const int ct = e.col_type ? e.col_type : d.ret;
        if (all_literal || is_null) {
            const uint64_t v = is_null ? DT_FN_NULL : dt_date_fn(d.fn, arg, img[0], img[1]);
            const int k = v == DT_FN_NULL ? add_const(0, true) : add_const(host_cast_prim(v, d.ret, ct), false);
            if (k < 0) return false;
            depth++;
            return emit(OP_CONST, (uint8_t)k);
        }
        for (size_t i = 0; i < nv; i++) {
            const HExpr& c = e.ch[v0 + i];
            if (!expr(c, depth) || !cast(c.col_type, d.arg_prim)) return false;
            if (d.fn == DF_DATEDIFF && !cast(BK_DATE, BK_TIMESTAMP)) return false;
        }
        depth = d0 + 1;
        return emit(OP_DATEFN, d.fn, (uint8_t)arg, (uint8_t)nv) && cast(d.ret, ct);
    }
    bool common_fn(const HExpr& e, int& depth) {
        if (const DateFnDef* d = date_fn_def(e.name)) return date_fn(e, *d, depth);
        const int d0 = depth;
        const int ct = e.col_type;
        if (e.name == "if") {
            if (!expr(e.ch[0], depth) || !to_bool(e.ch[0]) || !branch(e.ch[1], ct, depth) || !branch(e.ch[2], ct, depth)) return false;
            depth = d0 + 1;
            return emit(OP_SELECT);
        }
        if (e.name == "ifnull") {
            if (!branch(e.ch[0], ct, depth) || !branch(e.ch[1], ct, depth)) return false;
            depth = d0 + 1;
            return emit(OP_IFNULL);
        }
        if (e.name == "case_when") {   // WHEN c1 THEN t1 ... [ELSE e]  ==  if(c1, t1, if(c2, t2, ... e | NULL))
            const size_t n = e.ch.size(), pairs = n / 2;
            for (size_t i = 0; i < pairs; i++)
                if (!expr(e.ch[2 * i], depth) || !to_bool(e.ch[2 * i]) || !branch(e.ch[2 * i + 1], ct, depth)) return false;
            if (n % 2 == 1) { if (!branch(e.ch[n - 1], ct, depth)) return false; }
            else { int k = add_const(0, true); if (k < 0 || !emit(OP_CONST, (uint8_t)k)) return false; depth++; }
            if (depth > STACK_DEPTH - 1) return in->fail(BKGPU_EUNSUPPORTED, "CASE with %zu branches exceeds the device stack", pairs);
            for (size_t i = 0; i < pairs; i++) if (!emit(OP_SELECT)) return false;
            depth = d0 + 1;
            return true;
        }
        if (e.name == "pi") {
            const double pi = 3.14159265358979323846; uint64_t b; memcpy(&b, &pi, 8);
            int k = add_const(b, false); if (k < 0) return false;
            depth++;
            return emit(OP_CONST, (uint8_t)k) && cast(BK_DOUBLE, ct);
        }
        if (const int m2 = math2_fn(e.name); m2 >= 0) {   // arguments read with get_numberic<double>(); greatest / least fold left to right
            if (!expr(e.ch[0], depth) || !cast(e.ch[0].col_type, BK_DOUBLE)) return false;
            for (size_t i = 1; i < e.ch.size(); i++) {
                if (!expr(e.ch[i], depth) || !cast(e.ch[i].col_type, BK_DOUBLE) || !emit(OP_MATH2, (uint8_t)m2)) return false;
                depth--;
            }
            depth = d0 + 1;
            return cast(BK_DOUBLE, ct);
        }
        if (!expr(e.ch[0], depth)) return false;
        const int at = e.ch[0].col_type;
        if (e.name == "bit_count") return cast(at, BK_UINT64) && emit(OP_MATH, MF_BIT_COUNT) && cast(BK_INT64, ct);
        if (e.name == "cast_to_signed") return cast(at, BK_INT64) && cast(BK_INT64, ct);
        if (e.name == "cast_to_unsigned") return cast(at, BK_UINT64) && cast(BK_UINT64, ct);
        if (e.name == "cast_to_double") return cast(at, BK_DOUBLE) && cast(BK_DOUBLE, ct);
        if (!cast(at, BK_DOUBLE)) return false;   // get_numberic<double>()
        if (e.name == "abs") return emit(OP_MATH, MF_ABS) && cast(BK_DOUBLE, ct);
        if (e.name == "floor") return emit(OP_MATH, MF_FLOOR) && emit(OP_CAST, (uint8_t)BK_DOUBLE, (uint8_t)BK_INT64) && cast(BK_INT64, ct);
        if (e.name == "ceil" || e.name == "ceiling") return emit(OP_MATH, MF_CEIL) && emit(OP_CAST, (uint8_t)BK_DOUBLE, (uint8_t)BK_INT64) && cast(BK_INT64, ct);
        if (e.name == "sign") return emit(OP_MATH, MF_SIGN) && cast(BK_INT64, ct);
        if (const int m1 = math1_fn(e.name); m1 >= 0) return emit(OP_MATH, (uint8_t)m1) && cast(BK_DOUBLE, ct);
        if (e.name == "round") {
            int bits = 0;
            if (e.ch.size() == 2) {   // input[1].get_numberic<int>() of the literal (cast to its col_type first, literal.h:204-206)
                const HExpr& l = e.ch[1];
                uint64_t img = l.col_type ? host_cast_prim(l.lit_bits, l.lit_prim, l.col_type) : l.lit_bits;
                bits = (int)(int64_t)host_cast_prim(img, l.col_type ? l.col_type : l.lit_prim, BK_INT32);
            }
            const double base = std::pow(10.0, bits);
            uint64_t bb; memcpy(&bb, &base, 8);
            int k = add_const(bb, false); if (k < 0) return false;
            return emit(OP_MATH, MF_ROUND, (uint8_t)k) && cast(BK_DOUBLE, ct);
        }
        return in->fail(BKGPU_EUNSUPPORTED, "function '%s'", e.name.c_str());
    }
    // children of logical predicates are read with get_numberic<bool>() (predicate.h:31)
    bool to_bool(const HExpr& c) { return c.col_type == BK_BOOL ? true : emit(OP_CAST, (uint8_t)c.col_type, (uint8_t)BK_BOOL); }
    bool out_reg(int r) { return emit(OP_OUT, (uint8_t)r); }
    // the conjunction of `conj` as output `reg`; `where` names the conjuncts in the refusal of more than 8
    bool predicate(const std::vector<const HExpr*>& conj, int reg, const std::string& where = "") {
        if (!at_most_8_conjuncts(*in, conj.size(), where)) return false;
        for (auto* c : conj) { int depth = 0; if (!expr(*c, depth) || !to_bool(*c)) return false; }
        if (conj.size() > 1 && !emit(OP_AND, (uint8_t)conj.size())) return false;
        return out_reg(reg);
    }
};

static std::string expr_key(const HExpr& e) {  // structural identity, for lane sharing
    char buf[96];
    snprintf(buf, sizeof buf, "(%d:%d:%d_%d:%d:%llx", e.node_type, e.col_type, e.tuple_id, e.slot_id, e.fn_op, (unsigned long long)e.lit_bits);
    std::string s = buf;
    if (e.node_type == BK_FUNCTION_CALL && e.fn_op == BK_FT_COMMON) s += ":" + e.name;   // year(d) is not month(d)
    if (e.lit_prim == BK_STRING) s += ":'" + e.lit_str + "'";                            // nor is extract('year', d) extract('month', d)
    for (auto& c : e.ch) s += expr_key(c);
    return s + ")";
}
static void expr_cols(const HExpr& e, const Compiled& c, int& mask) {
    if (e.node_type == BK_SLOT_REF)
        for (size_t i = 0; i < c.cols.size(); i++) if (c.cols[i].tuple_id == e.tuple_id && c.cols[i].slot_id == e.slot_id) mask |= 1 << i;
    for (auto& ch : e.ch) expr_cols(ch, c, mask);
}
// can the expression yield NULL although every column it reads is valid?
static bool expr_makes_null(const HExpr& e) {
    if (e.node_type == BK_NULL_LITERAL) return true;
    if (e.node_type == BK_IS_NULL_PREDICATE || e.node_type == BK_IS_TRUE_PREDICATE) return false;
    if (e.node_type == BK_FUNCTION_CALL && (e.fn_op == BK_FT_DIVIDES || e.fn_op == BK_FT_MOD)) return true;
    if (e.node_type == BK_FUNCTION_CALL && e.fn_op == BK_FT_COMMON && e.name == "case_when" && e.ch.size() % 2 == 0) return true;
    if (e.node_type == BK_FUNCTION_CALL && e.fn_op == BK_FT_COMMON)
        if (const DateFnDef* d = date_fn_def(e.name))   // NULL for a date boost rejects, and for an unknown extract unit
            if (d->fn == DF_DAYOFWEEK || d->fn == DF_WEEKDAY || d->fn == DF_DAYOFYEAR || d->fn == DF_WEEK || d->fn == DF_YEARWEEK ||
                d->fn == DF_WEEKOFYEAR || d->fn == DF_EXTRACT) return true;
    if (e.node_type == BK_IN_PREDICATE) for (size_t i = 1; i < e.ch.size(); i++) if (e.ch[i].lit_null) return true;
    for (auto& c : e.ch) if (expr_makes_null(c)) return true;
    return false;
}

static int key_value_bits(int prim) {
    switch (prim) {
        case BK_INT64: case BK_UINT64: case BK_DOUBLE: case BK_DATETIME: case BK_FLOAT: return 64;  // FLOAT keys travel as their double image
        default: return 32;
    }
}

static const HNode* skip_passthrough(const HNode* n, bool* under_packet) {
    while (n && (n->node_type == BK_PACKET_NODE || n->node_type == BK_SELECT_MANAGER_NODE)) {
        if (n->node_type == BK_PACKET_NODE && under_packet) *under_packet = true;
        n = n->ch.empty() ? nullptr : &n->ch[0];
    }
    return n;
}

static bool lower_agg(Infer& in, Compiled& out, const HNode& agg, const std::vector<const HExpr*>& conjuncts, int scan_tuple, bool under_packet, bool allow_direct) {
    out.kind = PK_AGG;
    out.scan_tuple = scan_tuple;
    out.is_merge = agg.node_type == BK_MERGE_AGG_NODE;
    out.emit_default = agg.group_exprs.empty() && (under_packet || out.is_merge);
    out.agg_limit = agg.limit;
    if (agg.group_exprs.size() > MAX_GROUP) return in.fail(BKGPU_EUNSUPPORTED, "more than %d GROUP BY expressions", MAX_GROUP);
    if (agg.agg_fns.size() > MAX_AGG) return in.fail(BKGPU_EUNSUPPORTED, "more than %d aggregate functions", MAX_AGG);
    Program& p = out.prog; memset(&p, 0, sizeof p);
    AggPlan& ap = out.ap; memset(&ap, 0, sizeof ap); out.n_rb = 0;
    Lower lw{&out, &in, &p};
    int reg = 0, depth = 0;
    // ---- predicate: all conjuncts non-NULL true (filter_node.cpp:726-734) ----
    ap.pred_out = -1;
    if (out.is_merge && !conjuncts.empty()) return in.fail(BKGPU_EUNSUPPORTED, "filter below MERGE_AGG_NODE");
    bool any_distinct = false;
    for (auto& f : agg.agg_fns) any_distinct = any_distinct || f.distinct;   // (a distinct aggregate is never "initial": is_initialize, agg_fn_call.cpp:322-328)
    if (out.is_merge && agg.group_exprs.empty() && !agg.agg_fns.empty() && !any_distinct) {
        // a scalar merger skips input rows whose aggregates are all still "initial" (AggFnCall::all_is_initialize,
        // agg_node.cpp:519-522): pass = OR_k (count_k <> 0 | value_k IS NOT NULL), three-valued, NULL = skip
        for (size_t k = 0; k < agg.agg_fns.size(); k++) {
            const HExpr& f = agg.agg_fns[k];
            const int st = in.slot_type(f.tuple_id, f.inter_slot);
            if (st == BK_INVALID_TYPE) return in.fail(BKGPU_EINVAL, "MERGE_AGG: slot %d_%d is not declared", f.tuple_id, f.inter_slot);
            const int ci = lw.intern_col(f.tuple_id, f.inter_slot, st);
            if (ci >= MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
            if (!lw.emit(OP_LOAD_COL, (uint8_t)ci, st == BK_STRING ? 1 : st == BK_HLL ? 4 : 0, 0)) return false;
            if (f.name == "count" || f.name == "count_star") {
                const int z = lw.add_const(0, false); if (z < 0) return false;
                if (!lw.emit(OP_CONST, (uint8_t)z) || !lw.emit(OP_CMP, (uint8_t)BK_FT_NE, (uint8_t)host_prim_class(st))) return false;
            } else if (!lw.emit(OP_IS_NULL) || !lw.emit(OP_NOT3)) return false;
            if (k > 0 && !lw.emit(OP_OR, 2)) return false;
        }
        ap.pred_out = reg;
        if (!lw.out_reg(reg++)) return false;
    }
    if (!conjuncts.empty()) {
        ap.pred_out = reg;
        if (!lw.predicate(conjuncts, reg++)) return false;
    }
    // ---- group keys ----
    ap.n_group = (int)agg.group_exprs.size();
    int n_words = 0, half_word = -1;  // half_word: a word holding one 32-bit field (upper half free)
    for (int g = 0; g < ap.n_group; g++) {
        const HExpr& e = agg.group_exprs[(size_t)g];
        if (e.col_type == BK_STRING) return in.fail(BKGPU_EUNSUPPORTED, "GROUP BY over a STRING key is outside the GPU path");
        depth = 0;
        if (!lw.expr(e, depth)) return false;
        ap.key_out[g] = (uint8_t)reg; ap.key_prim[g] = (uint8_t)e.col_type;
        if (!lw.out_reg(reg++)) return false;
        int bits = key_value_bits(e.col_type);
        ap.key_bits[g] = (uint8_t)bits;
        if (bits == 64) { ap.key_word[g] = (uint8_t)n_words++; ap.key_shift[g] = 0; }
        else if (half_word >= 0) { ap.key_word[g] = (uint8_t)half_word; ap.key_shift[g] = 32; half_word = -1; }
        else { ap.key_word[g] = (uint8_t)n_words; ap.key_shift[g] = 0; half_word = n_words++; }
    }
    if (ap.n_group > 0) {  // null flags: one bit per group expression (encode_exprs_key's null-flag byte)
        int w, sh;
        if (half_word >= 0) { w = half_word; sh = 32; } else { w = n_words++; sh = 0; }
        for (int g = 0; g < ap.n_group; g++) { ap.key_null_word[g] = (uint8_t)w; ap.key_null_shift[g] = (uint8_t)(sh + g); }
    }
    if (n_words > MAX_KEYW) return in.fail(BKGPU_EUNSUPPORTED, "GROUP BY key wider than %d words", MAX_KEYW);
    ap.n_keyw = n_words;
    // ---- aggregates and lanes ----
    ap.n_agg = (int)agg.agg_fns.size();
    const int n_visible = ap.n_agg;
    int n_hidden = 0;
    ap.n_lanes = 1; ap.lane_op[0] = LN_ADD_I64;
    std::map<std::string, int> cnt_lane_of, acc_lane_of, arg_reg_of;
    out.arg_cols_mask.assign((size_t)MAX_AGG, 0);
    out.arg_can_null.assign((size_t)MAX_AGG, false);
    auto new_lane = [&](uint8_t op) -> int {
        if (ap.n_lanes >= MAX_LANES) { in.fail(BKGPU_EUNSUPPORTED, "more than %d accumulator lanes", MAX_LANES); return -1; }
        ap.lane_op[ap.n_lanes] = op; return ap.n_lanes++;
    };
    for (int k = 0; k < ap.n_agg; k++) {
        const HExpr& f = agg.agg_fns[(size_t)k];
        AggSpec& a = ap.agg[k]; memset(&a, 0, sizeof a);
        a.arg_out = 0xFF; a.out_prim = (uint8_t)f.col_type;
        if (out.is_merge && !f.distinct && f.name == "hll_add_agg") {
            // MERGE_AGG_NODE over the stores' RAW sketches (AggFnCall::merge -> hll_merge_agg, hll_common.cpp:630-703): register-wise max
            const int st = in.slot_type(f.tuple_id, f.inter_slot);
            if (st != BK_HLL) return in.fail(BKGPU_EUNSUPPORTED, "MERGE_AGG: hll_add_agg over an intermediate slot of type %d (a RAW HLL sketch is merged)", st);
            const int ci = lw.intern_col(f.tuple_id, f.inter_slot, BK_HLL);
            if (ci >= MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
            out.arg_cols_mask[(size_t)k] = 1 << ci;
            if (!lw.emit(OP_LOAD_COL, (uint8_t)ci, 4, 0)) return false;   // (the row: the merge reads the value's 16400 bytes itself)
            a.arg_out = (uint8_t)reg; a.nullable = 1;
            if (!lw.out_reg(reg++)) return false;
            a.kind = AG_HLL; a.arg_prim = BK_HLL; a.hll_col = (uint8_t)ci;
            const int l = new_lane(LN_HLL); if (l < 0) return false;
            a.acc_lane = (uint8_t)l;
            ap.n_hll++;
            continue;
        }
        if (out.is_merge && f.name == "rb_build_agg")
            return in.fail(BKGPU_EUNSUPPORTED, "MERGE_AGG of rb_build_agg is outside the GPU path: its input would be the stores' variable-length bitmaps");
        if (out.is_merge && !f.distinct) {
            // MERGE_AGG_NODE: the input rows carry the stores' intermediate slots; AggFnCall::merge (agg_fn_call.cpp:719-822)
            // adds counts and sums, folds MIN/MAX, and adds both halves of an AVG blob.  NULL intermediates are skipped.
            const int st = in.slot_type(f.tuple_id, f.inter_slot);
            if (st == BK_INVALID_TYPE) return in.fail(BKGPU_EINVAL, "MERGE_AGG: slot %d_%d is not declared", f.tuple_id, f.inter_slot);
            const bool blob = f.name == "avg";
            if (blob != (st == BK_STRING)) return in.fail(BKGPU_EUNSUPPORTED, "MERGE_AGG: %s over an intermediate slot of type %d", f.name.c_str(), st);
            const int ci = lw.intern_col(f.tuple_id, f.inter_slot, st);
            if (ci >= MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
            out.arg_cols_mask[(size_t)k] = 1 << ci;
            if (!lw.emit(OP_LOAD_COL, (uint8_t)ci, blob ? 1 : 0, 0)) return false;
            a.arg_out = (uint8_t)reg; a.nullable = 1;
            if (!lw.out_reg(reg++)) return false;
            const uint8_t cls = (uint8_t)(blob ? VC_F64 : host_prim_class(st));
            a.vclass = a.arg_vclass = cls;
            uint8_t op = cls == VC_F64 ? LN_ADD_F64 : LN_ADD_I64;
            if (blob) {
                a.kind = AG_AVG;
                if (n_visible + n_hidden >= MAX_AGG) return in.fail(BKGPU_EUNSUPPORTED, "more than %d aggregate accumulators", MAX_AGG);
                const int hk = n_visible + n_hidden++;
                AggSpec& h = ap.agg[hk]; memset(&h, 0, sizeof h);
                h.kind = AG_COUNT_MERGE; h.hidden = 1; h.vclass = h.arg_vclass = VC_I64; h.nullable = 1; h.acc_owner = 1;
                out.arg_cols_mask[(size_t)hk] = 1 << ci;
                if (!lw.emit(OP_LOAD_COL, (uint8_t)ci, 2, 0)) return false;
                h.arg_out = (uint8_t)reg;
                if (!lw.out_reg(reg++)) return false;
                int hl = new_lane(LN_ADD_I64); if (hl < 0) return false;
                h.acc_lane = (uint8_t)hl;
                a.cnt_lane = (uint8_t)hl; a.cnt_owner = 0;
            } else if (f.name == "count" || f.name == "count_star") {
                a.kind = AG_COUNT_MERGE; a.vclass = VC_I64; op = LN_ADD_I64;
            } else {
                if (f.name == "sum") a.kind = AG_SUM;
                else {
                    const bool mn = f.name == "min";
                    a.kind = mn ? AG_MIN : AG_MAX;
                    op = cls == VC_F64 ? (mn ? LN_MIN_F64 : LN_MAX_F64) : (cls == VC_U64 ? (mn ? LN_MIN_U64 : LN_MAX_U64) : (mn ? LN_MIN_I64 : LN_MAX_I64));
                }
                int cl = new_lane(LN_ADD_I64); if (cl < 0) return false;
                a.cnt_lane = (uint8_t)cl; a.cnt_owner = 1;
            }
            int al = new_lane(op); if (al < 0) return false;
            a.acc_lane = (uint8_t)al; a.acc_owner = 1;
            continue;
        }
        if (f.name == "count_star") { a.kind = AG_COUNT_STAR; continue; }
        if (f.ch.empty()) return in.fail(BKGPU_EINVAL, "%s() without an argument", f.name.c_str());
        if (f.ch.size() > 1) return in.fail(BKGPU_EUNSUPPORTED, "%s() with %zu arguments", f.name.c_str(), f.ch.size());
        const HExpr& arg = f.ch[0];
        // COUNT(non-null literal) is COUNT(*) (agg_fn_call.cpp:246-250)
        if (f.name == "count" && is_literal_node(arg.node_type) && !arg.lit_null) { a.kind = AG_COUNT_STAR; continue; }
        if (f.name == "hll_add_agg") {
            // the value lane references the group's sketch (AG_HLL); no counter, no lane shared with another aggregate
            a.kind = AG_HLL; a.arg_prim = (uint8_t)arg.col_type; a.nullable = 1;
            const int st = arg.node_type == BK_SLOT_REF ? in.slot_type(arg.tuple_id, arg.slot_id) : BK_INVALID_TYPE;
            const bool raw_f32 = arg.node_type == BK_SLOT_REF && arg.col_type == BK_FLOAT && (st == BK_FLOAT || st == BK_INVALID_TYPE);
            const std::string hkey = expr_key(arg) + (raw_f32 ? "#f32" : "");
            if (!arg_reg_of.count(hkey)) {
                if (raw_f32) {   // the column's own 4 bytes (OP_LOAD_COL b = 3), which the reference hashes
                    const int ci = lw.intern_col(arg.tuple_id, arg.slot_id, BK_FLOAT);
                    if (ci >= MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
                    if (!lw.emit(OP_LOAD_COL, (uint8_t)ci, 3, (uint8_t)out.col_side[(size_t)ci])) return false;
                } else { depth = 0; if (!lw.expr(arg, depth)) return false; }
                arg_reg_of[hkey] = reg;
                if (!lw.out_reg(reg++)) return false;
            }
            a.arg_out = (uint8_t)arg_reg_of[hkey];
            a.arg_vclass = (uint8_t)(raw_f32 ? VC_U64 : host_prim_class(arg.col_type));
            int m = 0; expr_cols(arg, out, m); out.arg_cols_mask[(size_t)k] = m; out.arg_can_null[(size_t)k] = expr_makes_null(arg);
            const int l = new_lane(LN_HLL); if (l < 0) return false;
            a.acc_lane = (uint8_t)l;
            ap.n_hll++;
            continue;
        }
        if (f.name == "rb_build_agg") {
            // no lane: each non-NULL value appends a (slot, rb_idx, low 32 bits) key to the pair buffer, which rb.cu turns into the bitmaps
            if (out.n_rb >= MAX_RB) return in.fail(BKGPU_EUNSUPPORTED, "more than %d rb_build_agg in one aggregate is outside the GPU path", MAX_RB);
            a.kind = AG_RB; a.arg_prim = (uint8_t)arg.col_type; a.nullable = 1; a.rb_idx = (uint8_t)out.n_rb++;
            a.acc_lane = a.cnt_lane = 0xFF;
            const std::string rkey = expr_key(arg);
            if (!arg_reg_of.count(rkey)) {
                depth = 0;
                if (!lw.expr(arg, depth)) return false;
                arg_reg_of[rkey] = reg;
                if (!lw.out_reg(reg++)) return false;
            }
            a.arg_out = (uint8_t)arg_reg_of[rkey];
            a.arg_vclass = (uint8_t)host_prim_class(arg.col_type);
            int m = 0; expr_cols(arg, out, m); out.arg_cols_mask[(size_t)k] = m; out.arg_can_null[(size_t)k] = expr_makes_null(arg);
            continue;
        }
        std::string key = expr_key(arg);
        if (!arg_reg_of.count(key)) {
            depth = 0;
            if (!lw.expr(arg, depth)) return false;
            arg_reg_of[key] = reg;
            if (!lw.out_reg(reg++)) return false;
        }
        a.arg_out = (uint8_t)arg_reg_of[key];
        a.arg_vclass = (uint8_t)host_prim_class(arg.col_type);
        a.nullable = 1;
        int m = 0; expr_cols(arg, out, m); out.arg_cols_mask[(size_t)k] = m; out.arg_can_null[(size_t)k] = expr_makes_null(arg);
        if (!cnt_lane_of.count(key)) { int l = new_lane(LN_ADD_I64); if (l < 0) return false; cnt_lane_of[key] = l; a.cnt_owner = 1; }
        a.cnt_lane = (uint8_t)cnt_lane_of[key];
        uint8_t op;
        if (f.name == "count") { a.kind = AG_COUNT; continue; }
        else if (f.name == "sum") { a.kind = AG_SUM; a.vclass = (uint8_t)host_prim_class(f.col_type); op = a.vclass == VC_F64 ? LN_ADD_F64 : LN_ADD_I64; }
        else if (f.name == "avg") { a.kind = AG_AVG; a.vclass = VC_F64; op = LN_ADD_F64; }
        else {
            bool mn = f.name == "min";
            a.kind = mn ? AG_MIN : AG_MAX; a.vclass = a.arg_vclass;
            op = a.vclass == VC_F64 ? (mn ? LN_MIN_F64 : LN_MAX_F64) : (a.vclass == VC_U64 ? (mn ? LN_MIN_U64 : LN_MAX_U64) : (mn ? LN_MIN_I64 : LN_MAX_I64));
        }
        std::string akey = key + "#" + std::to_string((int)op) + "#" + std::to_string((int)a.vclass);
        if (!acc_lane_of.count(akey)) { int l = new_lane(op); if (l < 0) return false; acc_lane_of[akey] = l; a.acc_owner = 1; }
        a.acc_lane = (uint8_t)acc_lane_of[akey];
    }
    ap.n_agg = n_visible + n_hidden;
    out.arg_cols_mask.resize((size_t)ap.n_agg); out.arg_can_null.resize((size_t)ap.n_agg);
    p.n_out = reg;
    if (reg > MAX_GROUP + MAX_AGG + 1) return in.fail(BKGPU_EUNSUPPORTED, "too many program outputs");
    // ---- output schema ----
    for (int g = 0; g < ap.n_group; g++) {
        const HExpr& e = agg.group_exprs[(size_t)g];
        bool sr = e.node_type == BK_SLOT_REF;
        out.out_cols.push_back({sr ? e.tuple_id : -1, sr ? e.slot_id : g, e.col_type, 0});
    }
    for (int k = 0; k < n_visible; k++) {
        const HExpr& f = agg.agg_fns[(size_t)k];
        int ft = in.slot_type(f.tuple_id, f.final_slot);
        if (ft == BK_INVALID_TYPE || ft == BK_STRING) ft = f.col_type;
        if (ap.agg[k].kind == AG_HLL) ft = BK_HLL;
        if (ap.agg[k].kind == AG_RB) ft = BK_BITMAP;
        out.out_cols.push_back({f.tuple_id, f.final_slot, ft, ap.agg[k].kind == AG_HLL ? 2 : ap.agg[k].kind == AG_RB ? 3 : 0});
        ap.agg[k].out_prim = (uint8_t)ft;
        if (ap.agg[k].kind == AG_AVG) out.out_cols.push_back({f.tuple_id, f.inter_slot != f.final_slot ? f.inter_slot : -1, BK_STRING, 1});
    }
    // ---- "direct" shape detection ----
    out.has_direct = false;
    DirectPlan& d = out.direct; memset(&d, 0, sizeof d); memset(d.agg_val, 0xFF, sizeof d.agg_val);
    do {
        std::vector<int> order;  // cols indices in [terms][key][values] order
        if (!allow_direct || out.is_merge || ap.n_hll || out.n_rb) break;
        if (!conjuncts.empty()) {
            if (conjuncts.size() > 2) break;
            bool ok = true;
            for (auto* cp : conjuncts) {
                const HExpr& c = *cp;
                if (c.node_type != BK_FUNCTION_CALL || c.fn_op < BK_FT_EQ || c.fn_op > BK_FT_LE || c.ch.size() != 2 || c.col_type != BK_BOOL) { ok = false; break; }
                const HExpr *col = &c.ch[0], *lit = &c.ch[1]; int op = c.fn_op;
                if (is_literal_node(col->node_type) && lit->node_type == BK_SLOT_REF) {
                    std::swap(col, lit);
                    op = op == BK_FT_GT ? BK_FT_LT : op == BK_FT_LT ? BK_FT_GT : op == BK_FT_GE ? BK_FT_LE : op == BK_FT_LE ? BK_FT_GE : op;
                }
                if (col->node_type != BK_SLOT_REF || !is_literal_node(lit->node_type) || lit->lit_null) { ok = false; break; }
                int at = c.arg_types[0];
                int st = in.slot_type(col->tuple_id, col->slot_id); if (st == BK_INVALID_TYPE) st = col->col_type;
                if (st != col->col_type) { ok = false; break; }
                int cc = host_prim_class(st), ac = host_prim_class(at);
                if ((cc == VC_F64) != (ac == VC_F64)) { ok = false; break; }  // would need an int<->double conversion per row
                if (is_datetime_family(at) && st != at) { ok = false; break; }   // (a change of type inside the family is a calendar conversion: generic path)
                if (lit->lit_prim == BK_STRING) { ok = false; break; }
                // Literal::get_value casts to its col_type, ScalarFnCall casts that to the arg type
                uint64_t bits = lit->col_type ? host_cast_prim(lit->lit_bits, lit->lit_prim, lit->col_type) : lit->lit_bits;
                bits = host_cast_prim(bits, lit->col_type ? lit->col_type : lit->lit_prim, at);
                DirectTerm& t = d.term[d.n_terms++];
                t.cmp = (uint8_t)op; t.vclass = (uint8_t)ac; t.cbits = bits;
                order.push_back(lw.intern_col(col->tuple_id, col->slot_id, st));
            }
            if (!ok) break;
        }
        if (ap.n_group > 1) break;
        if (ap.n_group == 1) {
            const HExpr& e = agg.group_exprs[0];
            if (e.node_type != BK_SLOT_REF) break;
            int st = in.slot_type(e.tuple_id, e.slot_id); if (st == BK_INVALID_TYPE) st = e.col_type;
            if (st != e.col_type || ap.n_keyw > 2) break;
            d.n_keys = 1;
            order.push_back(lw.intern_col(e.tuple_id, e.slot_id, st));
        }
        bool ok = true;
        std::vector<int> vals;
        for (int k = 0; k < ap.n_agg && ok; k++) {
            const HExpr& f = agg.agg_fns[(size_t)k];
            if (ap.agg[k].kind == AG_COUNT_STAR) continue;
            const HExpr& arg = f.ch[0];
            int st = arg.node_type == BK_SLOT_REF ? in.slot_type(arg.tuple_id, arg.slot_id) : BK_INVALID_TYPE;
            if (arg.node_type != BK_SLOT_REF || (st != BK_INVALID_TYPE && st != arg.col_type)) { ok = false; break; }
            int ci = lw.intern_col(arg.tuple_id, arg.slot_id, arg.col_type);
            size_t pos = 0;
            for (; pos < vals.size(); pos++) if (vals[pos] == ci) break;
            if (pos == vals.size()) vals.push_back(ci);
            d.agg_val[k] = (uint8_t)pos;
        }
        if (!ok || vals.size() > 4) break;
        {   // at most 3 lane operations per value column (ValOps)
            int ops[4] = {0, 0, 0, 0}; bool too_many = false;
            for (int k = 0; k < ap.n_agg; k++)
                if (ap.agg[k].kind != AG_COUNT_STAR && ap.agg[k].kind != AG_COUNT && ap.agg[k].acc_owner && ++ops[d.agg_val[k]] > 3) too_many = true;
            if (too_many) break;
        }
        d.n_vals = (int)vals.size();
        for (int v : vals) order.push_back(v);
        out.direct_cols = order;
        out.has_direct = true;
    } while (0);
    return true;
}

// ---------------------------------------------------------------- explain
static const char* op_name(int op) {
    static const char* n[] = {"END", "LOAD_COL", "CONST", "CAST", "CMP", "ARITH", "DIV_F64", "MOD", "BIT", "BIT_NOT", "NEG",
                              "LOGIC_NOT", "AND", "OR", "XOR", "NOT3", "IS_NULL", "IS_TRUE", "IN", "OUT", "SELECT", "IFNULL", "MATH", "MATH2", "DATEFN", "IN_SET"};
    return op >= 0 && op <= OP_IN_SET ? n[op] : "?";
}
// an IN set's shape (never its entries)
static std::string in_set_text(const InSet& s) {
    char buf[160];
    const size_t cap = s.image.size() - IN_SET_HEADER;
    snprintf(buf, sizeof buf, "distinct=%u capacity=%zu class=%d null=%d bytes=%zu", s.n_distinct, cap, s.vclass, (int)s.has_null, s.image.size() * 8);
    return buf;
}
// the window stages of a PK_WINDOW fragment (over a scan, or above an aggregate) and the query's ORDER BY above them
static void explain_window(const Compiled& c, std::string& s) {
    static const char* fn_names[] = {"count_star", "count", "sum", "avg", "min", "max", "row_number", "rank", "dense_rank", "percent_rank",
                                     "cume_dist", "ntile", "lead", "lag", "first_value", "last_value", "nth_value"};
    static const char* bound_names[] = {"PRECEDING", "FOLLOWING", "CURRENT ROW"};
    char buf[256];
    for (size_t k = 0; k < c.win.size(); k++) {
        const WinStage& w = c.win[k];
        snprintf(buf, sizeof buf, "window stage[%zu]: sort=%s keys=%zu partition=%d exprs=%zu fns=%zu", k, w.new_sort ? "new" : (w.sort_keys.empty() ? "none" : "shared"),
                 w.sort_keys.size(), w.n_part, w.exprs.size(), w.fns.size()); s += buf;
        if (w.has_frame) {
            auto bound = [&](const WinBound& b) {
                char t[48];
                if (b.unbounded) snprintf(t, sizeof t, "UNBOUNDED %s", bound_names[b.type]);
                else if (b.type == BK_BT_CURRENT_ROW) snprintf(t, sizeof t, "CURRENT ROW");
                else snprintf(t, sizeof t, "%lld %s", (long long)b.num, bound_names[b.type]);
                return std::string(t);
            };
            s += std::string(" frame=") + (w.frame_type == BK_FRAME_ROWS ? "ROWS " : "RANGE ") + bound(w.start) + " .. " + bound(w.end);
        }
        s += "\n";
        for (auto& sk : w.sort_keys) { snprintf(buf, sizeof buf, "  %s key: expr=%d prim=%d asc=%d\n", (&sk - w.sort_keys.data()) < w.n_part ? "partition" : "order", sk.out_reg, sk.prim, (int)sk.asc); s += buf; }
        for (auto& f : w.fns) { snprintf(buf, sizeof buf, "  fn %s -> %d_%d prim=%d arg=%d default=%d n=%lld method=%d\n", fn_names[f.kind], f.tuple_id, f.slot_id, f.out_prim, f.arg, f.def,
                                         (long long)f.n, f.method); s += buf; }
    }
    if (c.post) { snprintf(buf, sizeof buf, "post fragment above the window: kind=%d keys=%zu limit=%lld offset=%lld\n", c.post->kind, c.post->sort_keys.size(),
                           (long long)c.post->limit, (long long)c.post->offset); s += buf; }
}
static void explain(Compiled& c) {
    char buf[256];
    std::string& s = c.explain;
    snprintf(buf, sizeof buf, "kind=%d scan_tuple=%d cols=%zu\n", c.kind, c.scan_tuple, c.cols.size()); s += buf;
    for (size_t i = 0; i < c.cols.size(); i++) { snprintf(buf, sizeof buf, "  col[%zu] = %d_%d prim=%d\n", i, c.cols[i].tuple_id, c.cols[i].slot_id, c.cols[i].prim); s += buf; }
    for (size_t k = 0; k < c.dims.size(); k++) {
        const StarDim& d = c.dims[k];
        if (k == 0) { snprintf(buf, sizeof buf, "star: fact tuple=%d dims=%zu\n", c.scan_tuple, c.dims.size()); s += buf; }
        const ColRef &dk = c.cols[(size_t)d.key_col], &fk = c.cols[(size_t)d.fk_col];
        snprintf(buf, sizeof buf, "  dim[%zu] tuple=%d key=%d_%d fk=%d_%d cast=%d build_conjuncts=%d\n", k, d.tuple_id, dk.tuple_id, dk.slot_id, fk.tuple_id, fk.slot_id,
                 d.cast_prim, d.n_filter); s += buf;
    }
    if (c.kind == PK_AGG || c.kind == PK_JOIN_AGG || c.kind == PK_STAR_AGG) {
        const AggPlan& ap = c.ap;
        snprintf(buf, sizeof buf, "agg: n_group=%d n_keyw=%d n_agg=%d n_lanes=%d pred_out=%d direct=%d emit_default=%d\n", ap.n_group, ap.n_keyw,
                 ap.n_agg, ap.n_lanes, ap.pred_out, (int)c.has_direct, (int)c.emit_default); s += buf;
        for (int k = 0; k < ap.n_agg; k++) {
            const AggSpec& a = ap.agg[k];
            snprintf(buf, sizeof buf, "  agg[%d] kind=%d class=%d arg_class=%d acc_lane=%d cnt_lane=%d arg_out=%d out_prim=%d\n", k, a.kind, a.vclass,
                     a.arg_vclass, a.acc_lane, a.cnt_lane, a.arg_out, a.out_prim); s += buf;
            if (a.kind == AG_HLL && a.arg_prim == BK_HLL) {
                snprintf(buf, sizeof buf, "    hll_add_agg under MERGE_AGG: register-wise max of the RAW sketches of col[%d] (16400 bytes each)\n", a.hll_col); s += buf;
            } else if (a.kind == AG_HLL) {
                snprintf(buf, sizeof buf, "    hll_add_agg: arg_prim=%d hashes %d bytes%s (MurmurHash3_x64_128, seed 0x110) -> 16384 registers, RAW sketch of %d bytes\n",
                         a.arg_prim, hll_key_bytes(a.arg_prim), a.arg_vclass == VC_U64 && a.arg_prim == BK_FLOAT ? " of the FLOAT column" : "", HLL_RAW_BYTES); s += buf;
            } else if (a.kind == AG_RB) {
                snprintf(buf, sizeof buf, "    rb_build_agg: rb=%d arg_prim=%d adds the low 32 bits of the value -> pair key (slot << 34 | %d << 32 | value), "
                         "Roaring bitmap (runOptimize, portable serialization)\n", a.rb_idx, a.arg_prim, a.rb_idx); s += buf;
            }
        }
        if (c.has_direct) {
            for (int t = 0; t < c.direct.n_terms; t++) {
                snprintf(buf, sizeof buf, "  direct term[%d]: col=%d cmp=%d class=%d const=0x%llx\n", t, c.direct_cols[(size_t)t], c.direct.term[t].cmp,
                         c.direct.term[t].vclass, (unsigned long long)c.direct.term[t].cbits); s += buf;
            }
        }
    }
    if (c.kind == PK_SORT || c.kind == PK_FILTER) {
        snprintf(buf, sizeof buf, "rows: pred_out=%d limit=%lld offset=%lld direct=%d\n", c.ap.pred_out, (long long)c.limit, (long long)c.offset, (int)c.has_direct); s += buf;
        for (auto& k : c.sort_keys) { snprintf(buf, sizeof buf, "  order key: out=%d prim=%d asc=%d null_first=%d\n", k.out_reg, k.prim, (int)k.asc, (int)k.null_first); s += buf; }
    }
    if (c.kind == PK_WINDOW) {
        snprintf(buf, sizeof buf, "rows: pred_out=%d limit=%lld offset=%lld stages=%zu\n", c.ap.pred_out, (long long)c.limit, (long long)c.offset, c.win.size()); s += buf;
        explain_window(c, s);
    } else if (c.post && c.post->kind == PK_WINDOW) {
        const Compiled& w = *c.post;
        snprintf(buf, sizeof buf, "window stages above the aggregate: input columns=%zu having pred_out=%d limit=%lld offset=%lld stages=%zu\n", w.cols.size(),
                 w.ap.pred_out, (long long)w.limit, (long long)w.offset, w.win.size()); s += buf;
        explain_window(w, s);
    } else
    if (c.post) { snprintf(buf, sizeof buf, "post fragment above the aggregate: kind=%d keys=%zu pred_out=%d limit=%lld offset=%lld\n", c.post->kind, c.post->sort_keys.size(),
                           c.post->ap.pred_out, (long long)c.post->limit, (long long)c.post->offset); s += buf; }
    if (c.join_type == BK_FULL_JOIN) {
        const bool agg = c.kind == PK_JOIN_AGG;
        snprintf(buf, sizeof buf, "full join: k_join_pairs_full (the program below: the join conditions) -> gather -> %s; the filter above the join is the %s predicate (pred_out=%d)\n",
                 agg ? "aggregate over the joined row" : "sink", agg ? "aggregate's" : "sink's", agg ? c.jfast->ap.pred_out : c.post->ap.pred_out); s += buf;
    }
    if (c.n_build_filter || c.n_probe_filter) {
        snprintf(buf, sizeof buf, "child filters: build tuple=%d conjuncts=%d (once over the retained rows: multimap key validity, failing rows never in the tail); "
                 "probe tuple=%d conjuncts=%d (per probe batch: probe key validity)\n", c.build_tuple, c.n_build_filter, c.scan_tuple, c.n_probe_filter); s += buf;
    }
    if (c.apply_join_type) {
        snprintf(buf, sizeof buf, "apply: %s decorrelated into the join above; conjuncts moved from the subquery into the join conditions=%d, "
                 "folded from the filter above into the outer filter=%d\n", c.apply_join_type == BK_SEMI_JOIN ? "SEMI" : "ANTI_SEMI", c.apply_moved, c.apply_folded); s += buf;
    }
    if (c.sub) {   // the scalar subquery: its grouped aggregate, then the lookup that joins it to the outer rows
        if (c.sub->explain.empty()) explain(*c.sub);
        s += "scalar subquery: the subquery's aggregate grouped by its correlation keys {\n" + c.sub->explain + "}\n";
        for (size_t k = 0; k < c.sub_key_cols.size(); k++) {
            const ColRef& oc = c.cols[(size_t)c.sub_key_cols[k]];
            snprintf(buf, sizeof buf, "  lookup key[%zu]: outer col[%d] = %d_%d prim=%d cast=%d\n", k, c.sub_key_cols[k], oc.tuple_id, oc.slot_id, oc.prim,
                     c.sub->ap.key_prim[k]); s += buf;
        }
        for (size_t k = 0; k < c.sub_out_cols.size(); k++) {
            snprintf(buf, sizeof buf, "  lookup col[%d] <- subquery agg[%d] (no group: %s)\n", c.sub_out_cols[k], c.sub_out_agg[k],
                     c.sub->ap.agg[c.sub_out_agg[k]].kind <= AG_COUNT ? "0" : "NULL"); s += buf;
        }
        s += "  k_apply_lookup per outer batch, then the aggregate below over the outer columns and the looked-up ones\n";
    }
    snprintf(buf, sizeof buf, "program: %d instr, %d outputs\n", c.prog.n_instr, c.prog.n_out); s += buf;
    for (int i = 0; i < c.prog.n_instr; i++) {
        const Instr& in = c.prog.code[i];
        snprintf(buf, sizeof buf, "  %02d %-9s a=%d b=%d c=%d", i, op_name(in.op), in.a, in.b, in.c); s += buf;
        if (in.op == OP_CONST) { snprintf(buf, sizeof buf, "   ; 0x%llx%s", (unsigned long long)c.prog.cbits[in.a], ((c.prog.cnull >> in.a) & 1) ? " NULL" : ""); s += buf; }
        if (in.op == OP_IN_SET) s += "   ; set " + std::to_string(in.b) + ": " + in_set_text(c.in_sets->sets[in.b]);
        s += "\n";
    }
    if (c.in_sets && !c.in_sets->sets.empty()) {   // every set of the plan, whichever of its programs probes it
        size_t bytes = 0;
        for (auto& x : c.in_sets->sets) bytes += x.image.size() * 8;
        snprintf(buf, sizeof buf, "in sets: %zu, %zu bytes\n", c.in_sets->sets.size(), bytes); s += buf;
        for (size_t i = 0; i < c.in_sets->sets.size(); i++) s += "  set " + std::to_string(i) + ": " + in_set_text(c.in_sets->sets[i]) + "\n";
    }
}

void patch_in_sets(Compiled& c, const std::vector<uint64_t>& addr) {
    auto fix = [&](Program& q) {
        for (int i = 0; i < q.n_instr; i++) if (q.code[i].op == OP_IN_SET) q.cbits[q.code[i].a] = addr[q.code[i].b];
    };
    fix(c.prog);
    fix(c.build_filter); fix(c.probe_filter);
    for (StarDim& d : c.dims) fix(d.filter);
    for (WinStage& w : c.win) for (Program& q : w.exprs) fix(q);
    if (c.post) patch_in_sets(*c.post, addr);
    if (c.jfast) patch_in_sets(*c.jfast, addr);
    if (c.sub) patch_in_sets(*c.sub, addr);
}

// ---------------------------------------------------------------- steps shared by the fragments
static bool infer_node(Infer& in, HNode& n) {
    for (auto& e : n.conjuncts) if (!infer_expr(in, e)) return false;
    for (auto& e : n.group_exprs) if (!infer_expr(in, e)) return false;
    for (auto& e : n.agg_fns) if (!infer_expr(in, e)) return false;
    for (auto& e : n.order_exprs) if (!infer_expr(in, e)) return false;
    if (n.frame_start.has_expr && !infer_expr(in, n.frame_start.expr)) return false;
    if (n.frame_end.has_expr && !infer_expr(in, n.frame_end.expr)) return false;
    for (auto& c : n.ch) if (!infer_node(in, c)) return false;
    return true;
}

static std::vector<const HExpr*> conjuncts_of(const HNode* n) {
    std::vector<const HExpr*> v;
    if (n) for (auto& e : n->conjuncts) v.push_back(&e);
    return v;
}

// LIMIT n OFFSET m (LimitNode) over rows already capped at `limit` (-1 = none): the fragment keeps the first n + m rows and skips m of them
static void merge_limit(const HNode* limit_node, int64_t& limit, int64_t& offset) {
    if (!limit_node) return;
    offset = limit_node->offset;
    if (limit_node->limit >= 0) {   // (limit -1 = OFFSET only: every row is kept)
        const int64_t lim = limit_node->limit + limit_node->offset;
        if (limit < 0 || lim < limit) limit = lim;
    }
}

// the keys of a SORT node, one program output each from `reg` on
static bool lower_order_by(Lower& lw, const HNode& sort, std::vector<SortKey>& keys, int& reg) {
    if (sort.order_exprs.empty()) return lw.in->fail(BKGPU_EINVAL, "SORT node without order expressions");
    if (sort.order_exprs.size() > 4) return lw.in->fail(BKGPU_EUNSUPPORTED, "more than 4 ORDER BY expressions");
    for (size_t i = 0; i < sort.order_exprs.size(); i++) {
        const HExpr& e = sort.order_exprs[i];
        if (e.col_type == BK_STRING) return lw.in->fail(BKGPU_EUNSUPPORTED, "ORDER BY over a STRING key is outside the GPU path");
        int depth = 0;
        if (!lw.expr(e, depth)) return false;
        keys.push_back({reg, e.col_type, sort.is_asc[i] != 0, sort.is_null_first[i] != 0});
        if (!lw.out_reg(reg++)) return false;
    }
    return true;
}

// a filter node's conjunction as output `reg` (ap.pred_out; -1 without conjuncts)
static bool lower_predicate(Lower& lw, const HNode* filter, AggPlan& ap, int& reg) {
    ap.pred_out = -1;
    if (!filter || filter->conjuncts.empty()) return true;
    ap.pred_out = reg;
    return lw.predicate(conjuncts_of(filter), reg++);
}

// a one-output program of its own (a join child's or a star dimension's filter, a window expression): constants numbered from 0, the
// columns it reads become plan columns
template <class F> static bool lower_own_program(Infer& in, Compiled& out, Program& prog, F&& body) {
    memset(&prog, 0, sizeof prog);
    Lower l{&out, &in, &prog};
    if (!body(l)) return false;
    prog.n_out = 1;
    return true;
}

// every slot of `tuple_id` becomes a plan column and an output column, in the order of its descriptor
static bool intern_tuple(Infer& in, Compiled& out, Lower& lw, int tuple_id, const char* tuple_name, const char* row_name) {
    const HTuple* t = nullptr;
    for (auto& x : out.tuples) if (x.tuple_id == tuple_id) t = &x;
    if (!t || t->slots.empty()) return in.fail(BKGPU_EINVAL, "%s %d has no descriptor", tuple_name, tuple_id);
    for (auto& sl : t->slots) {
        if (prim_storage(sl.second) < 0 || sl.second == BK_STRING || sl.second == BK_HLL)
            return in.fail(BKGPU_EUNSUPPORTED, "column %d_%d has type %d: outside the GPU path", tuple_id, sl.first, sl.second);
        if (lw.intern_col(tuple_id, sl.first, sl.second) >= MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns in %s", MAX_COLS, row_name);
        out.out_cols.push_back({tuple_id, sl.first, sl.second, 0});
    }
    return true;
}

// A sink fragment (Compiled::post, kind PK_SORT / PK_FILTER) over another fragment's output rows: its "scan tuple" is `out.out_cols`, in
// order.  Above an aggregate ([LIMIT ->] [SORT ->] [HAVING ->]: SortNode::open src/exec/sort_node.cpp:278-346, FilterNode::get_next
// src/exec/filter_node.cpp:726-795 over the rows AggNode::get_next emits), the query's ORDER BY above window stages, and the joined rows
// of a join that returns them.
struct Sink {
    const HNode* sort;       // ORDER BY keys: PK_SORT, else PK_FILTER
    const HNode* pred;       // HAVING, or the filter above a FULL join (it judges the NULL-extended rows too)
    int64_t own_limit;       // without a SORT: the rows' own limit
    bool agg_rows;           // rows of an aggregate or a window: AVG blobs ride along as 16-byte payload columns, a column twice is refused
    const char* too_wide;    // refused: more than MAX_COLS input columns
    const char* outside;     // refused: a key or the predicate reads a column that is not an input column
};
static bool lower_sink(Infer& in, Compiled& out, const Sink& s, const HNode* limit_node) {
    if (out.out_cols.size() > (size_t)MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d %s", MAX_COLS, s.too_wide);
    auto post = std::make_shared<Compiled>();
    Compiled& pc = *post;
    pc.kind = s.sort ? PK_SORT : PK_FILTER;
    pc.tuples = out.tuples; pc.scan_tuple = -1; pc.in_sets = out.in_sets;
    Program& p = pc.prog; memset(&p, 0, sizeof p);
    memset(&pc.ap, 0, sizeof pc.ap);
    Lower lw{&pc, &in, &p};
    for (const OutCol& oc : out.out_cols) {
        const int prim = s.agg_rows && oc.kind == 1 ? BK_STRING : oc.prim;
        const int ci = lw.intern_col(oc.tuple_id, oc.slot_id, prim);
        if (s.agg_rows && ci != (int)pc.out_cols.size()) return in.fail(BKGPU_EUNSUPPORTED, "aggregate output columns %d_%d appear twice", oc.tuple_id, oc.slot_id);
        pc.out_cols.push_back({oc.tuple_id, oc.slot_id, prim, oc.kind});
    }
    int reg = 0;
    if (s.pred && s.pred->limit != -1 && s.sort) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a HAVING filter below a sort is order dependent");
    if (!lower_predicate(lw, s.pred, pc.ap, reg)) return false;
    pc.limit = s.sort ? s.sort->limit : s.own_limit;
    if (s.sort && !lower_order_by(lw, *s.sort, pc.sort_keys, reg)) return false;
    merge_limit(limit_node, pc.limit, pc.offset);
    p.n_out = reg;
    if (pc.cols.size() != out.out_cols.size()) return in.fail(BKGPU_EUNSUPPORTED, "%s", s.outside);
    pc.has_direct = false;
    out.post = post;
    return true;
}

// ---------------------------------------------------------------- SORT / filter-only fragments
// Rows of the scan tuple are returned (all slots of its tuple descriptor), ordered / filtered.
static bool lower_sort(Infer& in, Compiled& out, const HNode& sort, const HNode* filter, const HNode& scan) {
    out.kind = PK_SORT;
    out.scan_tuple = scan.tuple_id;
    out.limit = sort.limit;
    if (filter && filter->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a filter below a sort is order dependent");
    Program& p = out.prog; memset(&p, 0, sizeof p);
    memset(&out.ap, 0, sizeof out.ap);
    Lower lw{&out, &in, &p};
    if (!intern_tuple(in, out, lw, scan.tuple_id, "scan tuple", "the scan tuple")) return false;
    int reg = 0;
    if (!lower_predicate(lw, filter, out.ap, reg) || !lower_order_by(lw, sort, out.sort_keys, reg)) return false;
    p.n_out = reg;
    // direct shape: one plain column key, no filter (config C5)
    out.has_direct = false;
    if (!filter && sort.order_exprs.size() == 1 && sort.order_exprs[0].node_type == BK_SLOT_REF) {
        const HExpr& e = sort.order_exprs[0];
        int st = in.slot_type(e.tuple_id, e.slot_id);
        if (st == e.col_type && (prim_storage(st) == ST_I64 || prim_storage(st) == ST_U64 || prim_storage(st) == ST_F64 ||
                                 prim_storage(st) == ST_I32 || prim_storage(st) == ST_U32)) {
            out.has_direct = true;
            out.direct_cols = {lw.intern_col(e.tuple_id, e.slot_id, st)};
        }
    }
    return true;
}

static bool lower_filter(Infer& in, Compiled& out, const HNode* limit_node, const HNode& top, const HNode& scan) {
    out.kind = PK_FILTER;
    out.scan_tuple = scan.tuple_id;
    const HNode* filter = is_filter(&top) ? &top : nullptr;
    out.limit = filter ? filter->limit : scan.limit;   // FilterNode honours its own limit in input order (filter_node.cpp:786-791)
    out.offset = 0;
    merge_limit(limit_node, out.limit, out.offset);
    Program& p = out.prog; memset(&p, 0, sizeof p);
    memset(&out.ap, 0, sizeof out.ap);
    Lower lw{&out, &in, &p};
    if (!intern_tuple(in, out, lw, scan.tuple_id, "scan tuple", "the scan tuple")) return false;
    int reg = 0;
    if (!lower_predicate(lw, filter, out.ap, reg)) return false;
    p.n_out = reg;
    return true;
}

// ---------------------------------------------------------------- two-table joins
// The reference builds its hash map on the OUTER (driver) child and probes with the inner child's rows (JoinNode::hash_join,
// src/exec/join_node.cpp:920-1022; Joiner::construct_hash_map, src/exec/joiner.cpp:624-631); the key is the cast equal-slot value
// (strip_out_equal_slots, joiner.cpp:166-217).
static void intern_slots(Lower& lw, Infer& in, const HExpr& e) {   // every column `e` reads becomes a plan column
    if (e.node_type == BK_SLOT_REF) {
        const int st = in.slot_type(e.tuple_id, e.slot_id);
        lw.intern_col(e.tuple_id, e.slot_id, st == BK_INVALID_TYPE ? e.col_type : st);
    }
    for (auto& c : e.ch) intern_slots(lw, in, c);
}
static void expr_tuples(const HExpr& e, std::vector<int>& t) {
    if (e.node_type == BK_SLOT_REF && std::find(t.begin(), t.end(), e.tuple_id) == t.end()) t.push_back(e.tuple_id);
    for (auto& c : e.ch) expr_tuples(c, t);
}
// LEFT / SEMI / ANTI_SEMI: the filter of the child scanning `tuple_id` (FilterNode under JoinNode) stays that child's: a program of its own
// whose output 0 is the conjunction.  Its columns become plan columns.
static bool lower_child_filter(Infer& in, Compiled& out, const HNode* filt, int tuple_id, Program& prog, int& n) {
    memset(&prog, 0, sizeof prog); n = 0;
    if (!filt || filt->conjuncts.empty()) return true;
    const std::string where = " in the filter of join child " + std::to_string(tuple_id);
    if (!at_most_8_conjuncts(in, filt->conjuncts.size(), where)) return false;   // (before the check of the tuples it reads)
    for (auto& e : filt->conjuncts) {
        std::vector<int> ts; expr_tuples(e, ts);
        for (int t : ts) if (t != tuple_id) return in.fail(BKGPU_EINVAL, "the filter of join child %d reads tuple %d", tuple_id, t);
    }
    n = (int)filt->conjuncts.size();
    return lower_own_program(in, out, prog, [&](Lower& l) { return l.predicate(conjuncts_of(filt), 0, where); });
}
// the children, build (outer) side first, each [FILTER ->] SCAN.  RIGHT JOIN: the reference swaps the roles — the right child becomes the
// outer (preserved, driver) table (join_node.cpp:151-156) — and the join is lowered as LEFT.
static bool join_children(Infer& in, const HNode& join, int& jt, const HNode* side[2], const HNode* filt[2]) {
    for (int i = 0; i < 2; i++) {
        const HNode* c = skip_passthrough(&join.ch[(size_t)(jt == BK_RIGHT_JOIN ? 1 - i : i)], nullptr);
        filt[i] = nullptr;
        if (is_filter(c)) { filt[i] = c; c = c->ch.empty() ? nullptr : skip_passthrough(&c->ch[0], nullptr); }
        if (!c || c->node_type != BK_SCAN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "JOIN children must be [FILTER ->] SCAN");
        if (filt[i] && filt[i]->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT below a join is order dependent");
        side[i] = c;
    }
    if (jt == BK_RIGHT_JOIN) jt = BK_LEFT_JOIN;
    return true;
}
// the join key: the first build = probe slot equality among the join conditions; the others go to `rest` (residual conditions)
static bool join_equality(Infer& in, const HNode& join, int build_tuple, int probe_tuple, const HExpr*& bk, const HExpr*& pk, std::vector<const HExpr*>& rest) {
    bk = pk = nullptr;
    for (auto& e : join.conjuncts) {
        bool taken = false;
        if (!bk && e.node_type == BK_FUNCTION_CALL && e.fn_op == BK_FT_EQ && e.ch.size() == 2 && e.ch[0].node_type == BK_SLOT_REF && e.ch[1].node_type == BK_SLOT_REF) {
            const HExpr *a = &e.ch[0], *b = &e.ch[1];
            if (a->tuple_id == build_tuple && b->tuple_id == probe_tuple) { bk = a; pk = b; taken = true; }
            else if (b->tuple_id == build_tuple && a->tuple_id == probe_tuple) { bk = b; pk = a; taken = true; }
        }
        if (!taken) rest.push_back(&e);
    }
    return bk || in.fail(BKGPU_EUNSUPPORTED, "join without an equality between the two tables (nested loop) is outside the GPU path");
}
// the type the build / dimension key `a` and the probe / fact key `b` are compared in (strip_out_equal_slots' cast, joiner.cpp:166-217):
// equal types as they are, two signed types as INT64, two unsigned ones as UINT64; the reference compares any other pair as STRING
static bool join_key_cast(Infer& in, int a, int b, int& cast) {
    if (a == b) cast = a;
    else if (is_signed_t(a) && is_signed_t(b)) cast = BK_INT64;
    else if (is_uint_t(a) && is_uint_t(b)) cast = BK_UINT64;
    else return in.fail(BKGPU_EUNSUPPORTED, "join keys of types %d and %d are compared as STRING in the reference: outside the GPU path", a, b);
    if (cast == BK_STRING || is_double_t(cast)) return in.fail(BKGPU_EUNSUPPORTED, "join key type %d is outside the GPU path", cast);
    return true;
}

// The aggregate over the joined row (Compiled::jfast): the same aggregate lowered again with every column as a column of ONE (virtual,
// joined) tuple, build-side / dimension columns gathered to probe-row alignment first.  Its key words and lanes must be the main plan's and
// every column it reads one of the main plan's (jfast_of_main).  1 = lowered; 0 = it does not lower alike (`why`: its error); -1 = it
// reads `missing`, which is no main plan column.
static int lower_joined_row_agg(Compiled& out, const HNode& agg, const std::vector<const HExpr*>& conj, int scan_tuple, bool under_packet,
                                std::string& why, ColRef& missing) {
    auto jf = std::make_shared<Compiled>();
    jf->tuples = out.tuples; jf->build_tuple = -1; jf->in_sets = out.in_sets;
    Infer in2{}; in2.tuples = &jf->tuples;
    if (!lower_agg(in2, *jf, agg, conj, scan_tuple, under_packet, true) || memcmp(&jf->ap.n_keyw, &out.ap.n_keyw, sizeof(int32_t) * 4) != 0 ||
        jf->ap.n_lanes != out.ap.n_lanes) { why = in2.err; return 0; }
    std::vector<int> of_main;
    for (auto& c : jf->cols) {
        int m = -1;
        for (size_t i = 0; i < out.cols.size(); i++) if (out.cols[i].tuple_id == c.tuple_id && out.cols[i].slot_id == c.slot_id) m = (int)i;
        if (m < 0) { missing = c; return -1; }
        of_main.push_back(m);
    }
    out.jfast = jf;
    out.jfast_of_main = of_main;
    return 1;
}

// AGG over an equi-join (config C3).  Filters of both children and the residual join conditions become one predicate over the joined
// row — for an INNER join that is the same set of rows.  LEFT / SEMI / ANTI: a child's filter must remove the child's rows before the join
// (a build row that fails it would still come out of the ANTI tail, or NULL-extended), so each child's filter is a program of its own
// (Compiled::build_filter / probe_filter) and the main program keeps the residual conditions alone.
// FULL: the residual conditions decide the pairs (k_join_pairs_full); the filter above the join — the planner keeps a join FULL only under a
// NULL-tolerant one (join_node.cpp:171-203) — judges every emitted row, NULL-extended ones included, as the predicate of `jfast`, the
// aggregate over the pairs' gathered columns.
static bool lower_join_agg(Infer& in, Compiled& out, const HNode& agg, const HNode& join, bool under_packet, const HNode* above) {
    int jt = join.join_type;
    if (jt != BK_INNER_JOIN && jt != BK_LEFT_JOIN && jt != BK_RIGHT_JOIN && jt != BK_SEMI_JOIN && jt != BK_ANTI_SEMI_JOIN && jt != BK_FULL_JOIN)
        return in.fail(BKGPU_EUNSUPPORTED, "join type %d is outside the GPU path", jt);
    if (join.ch.size() != 2) return in.fail(BKGPU_EINVAL, "JOIN node needs two children");
    const HNode *side[2], *filt[2];
    if (!join_children(in, join, jt, side, filt)) return false;
    // the fused predicate (child filters + residual conditions over the joined row) equals filter-then-join only for INNER joins
    // a filter ABOVE the join sees the joined row: for an INNER join it simply joins the residual conditions; above an outer join it would also
    // have to judge the NULL-extended rows, after the match decision — a second predicate the probe does not carry
    const bool full = jt == BK_FULL_JOIN;
    if (full && (filt[0] || filt[1])) return in.fail(BKGPU_EUNSUPPORTED, "FULL join over filtered children is outside the GPU path");
    if (jt != BK_INNER_JOIN && !full && above) return in.fail(BKGPU_EUNSUPPORTED, "a filter between the aggregate and a LEFT / SEMI / ANTI join is outside the GPU path");
    // LEFT / SEMI / ANTI: a child's filter removes that child's rows before the join (lower_child_filter), except on the preserved side of LEFT
    if (jt == BK_LEFT_JOIN && filt[0]) return in.fail(BKGPU_EUNSUPPORTED, "a filter on the preserved side of a LEFT / RIGHT join is outside the GPU path");
    const int build_tuple = side[0]->tuple_id, probe_tuple = side[1]->tuple_id;
    out.build_tuple = build_tuple;
    std::vector<const HExpr*> conj;
    const HExpr *bk, *pk;
    if (!join_equality(in, join, build_tuple, probe_tuple, bk, pk, conj)) return false;
    if (jt == BK_INNER_JOIN) for (int i = 0; i < 2; i++) if (filt[i]) for (auto& e : filt[i]->conjuncts) conj.push_back(&e);
    std::vector<const HExpr*> above_conj;
    if (above) for (auto& e : above->conjuncts) (full ? above_conj : conj).push_back(&e);
    int cast;
    if (!join_key_cast(in, bk->col_type, pk->col_type, cast)) return false;
    if (full && agg.node_type == BK_MERGE_AGG_NODE) return in.fail(BKGPU_EUNSUPPORTED, "MERGE_AGG over a FULL join is outside the GPU path");
    if (!lower_agg(in, out, agg, conj, probe_tuple, under_packet, false)) return false;
    if (full) {   // the pairs kernel runs the main program for its predicate alone (the residual conditions): the aggregate is jfast's
        Program& q = out.prog;
        int n = 0;
        if (out.ap.pred_out >= 0) { while (n < q.n_instr && !(q.code[n].op == OP_OUT && q.code[n].a == out.ap.pred_out)) n++; n++; }
        q.n_instr = n; q.n_out = out.ap.pred_out >= 0 ? out.ap.pred_out + 1 : 0;
    }
    out.kind = PK_JOIN_AGG;
    out.join_type = jt; out.join_key_prim = cast;
    Program dummy; memset(&dummy, 0, sizeof dummy);
    Lower lw{&out, &in, &dummy};
    out.build_key_col = lw.intern_col(bk->tuple_id, bk->slot_id, in.slot_type(bk->tuple_id, bk->slot_id));
    out.probe_key_col = lw.intern_col(pk->tuple_id, pk->slot_id, in.slot_type(pk->tuple_id, pk->slot_id));
    for (auto* e : above_conj) intern_slots(lw, in, *e);   // (FULL: read by jfast's predicate alone, gathered like the aggregate's columns)
    if (jt != BK_INNER_JOIN && (!lower_child_filter(in, out, filt[0], build_tuple, out.build_filter, out.n_build_filter) ||
                                !lower_child_filter(in, out, filt[1], probe_tuple, out.probe_filter, out.n_probe_filter))) return false;
    if ((int)out.cols.size() > MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
    // INNER: the FK -> PK fast path, usable while every probe row has exactly one match.  FULL: the path itself, with the filter above the
    // join as the predicate
    if (jt == BK_INNER_JOIN || full) {
        std::string why; ColRef missing;
        if (lower_joined_row_agg(out, agg, full ? above_conj : conj, probe_tuple, under_packet, why, missing) <= 0 && full)
            return in.fail(BKGPU_EUNSUPPORTED, "the aggregate over the FULL join's row could not be lowered: %s", why.c_str());
    }
    return true;
}

// ---- star joins: AGG over a tree of INNER joins with 3 to 5 [FILTER ->] SCAN leaves ----
// The reference runs these as nested JoinNodes (a left-deep chain from JoinReorder, src/physical_plan/join_reorder.cpp:116-134).  For INNER
// joins the joined rows do not depend on the tree's shape, so left-deep, right-deep and bushy trees lower alike: the fact tuple is the leaf
// that has an equality with every other leaf, every other leaf is a dimension keyed by its first equality with the fact tuple.
static int join_leaves(const HNode* n) {
    n = skip_passthrough(n, nullptr);
    if (is_filter(n)) n = n->ch.empty() ? nullptr : skip_passthrough(&n->ch[0], nullptr);
    if (!n || n->node_type != BK_JOIN_NODE) return 1;
    int k = 0;
    for (auto& c : n->ch) k += join_leaves(&c);
    return k;
}
static bool star_walk(Infer& in, const HNode* n, std::vector<int>& leaves, std::vector<const HExpr*>& conds) {
    n = skip_passthrough(n, nullptr);
    if (is_filter(n)) {
        if (n->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a filter inside a join is order dependent: outside the GPU path");
        for (auto& e : n->conjuncts) conds.push_back(&e);
        n = n->ch.empty() ? nullptr : skip_passthrough(&n->ch[0], nullptr);
    }
    if (n && n->node_type == BK_JOIN_NODE) {
        if (n->join_type != BK_INNER_JOIN) return in.fail(BKGPU_EUNSUPPORTED, "join type %d in a join of more than two tables: only INNER joins are lowered", n->join_type);
        if (n->ch.size() != 2) return in.fail(BKGPU_EINVAL, "JOIN node needs two children");
        for (auto& e : n->conjuncts) conds.push_back(&e);
        return star_walk(in, &n->ch[0], leaves, conds) && star_walk(in, &n->ch[1], leaves, conds);
    }
    if (!n || n->node_type != BK_SCAN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "JOIN children must be [FILTER ->] SCAN or JOIN");
    leaves.push_back(n->tuple_id);
    return true;
}
static bool slot_eq(const HExpr& e) {
    return e.node_type == BK_FUNCTION_CALL && e.fn_op == BK_FT_EQ && e.ch.size() == 2 && e.ch[0].node_type == BK_SLOT_REF && e.ch[1].node_type == BK_SLOT_REF &&
           e.ch[0].tuple_id != e.ch[1].tuple_id;
}

static bool lower_star_agg(Infer& in, Compiled& out, const HNode& agg, const HNode& join, bool under_packet, const HNode* above) {
    std::vector<int> leaves; std::vector<const HExpr*> conds;
    if (!star_walk(in, &join, leaves, conds)) return false;
    if (leaves.size() > 5) return in.fail(BKGPU_EUNSUPPORTED, "a star join of %zu tables has more than 4 dimensions", leaves.size());
    if (above) for (auto& e : above->conjuncts) conds.push_back(&e);
    auto linked = [&](int a, int b) {
        for (auto* e : conds)
            if (slot_eq(*e) && ((e->ch[0].tuple_id == a && e->ch[1].tuple_id == b) || (e->ch[0].tuple_id == b && e->ch[1].tuple_id == a))) return true;
        return false;
    };
    int fact = -1;
    for (int t : leaves) {
        bool all = true;
        for (int u : leaves) if (u != t && !linked(t, u)) all = false;
        if (all) { fact = t; break; }
    }
    if (fact < 0) return in.fail(BKGPU_EUNSUPPORTED, "join of %zu tables without a star centre (a dimension keyed only to another dimension): outside the GPU path", leaves.size());
    std::vector<const HExpr*> taken;
    for (int t : leaves) {
        if (t == fact) continue;
        StarDim d; d.tuple_id = t;
        const HExpr *dk = nullptr, *fk = nullptr;
        for (auto* e : conds) {
            if (!slot_eq(*e)) continue;
            const HExpr *a = &e->ch[0], *b = &e->ch[1];
            if (a->tuple_id == fact && b->tuple_id == t) std::swap(a, b);
            if (a->tuple_id == t && b->tuple_id == fact) { dk = a; fk = b; taken.push_back(e); break; }
        }
        if (!join_key_cast(in, dk->col_type, fk->col_type, d.cast_prim)) return false;
        d.key_col = dk->slot_id; d.fk_col = fk->slot_id;   // (slot ids until the columns are interned below)
        out.dims.push_back(d);
    }
    // conjuncts over one dimension alone run once over its rows at build time; everything else is the aggregate's predicate
    std::vector<const HExpr*> conj;
    std::vector<std::vector<const HExpr*>> dim_conj(out.dims.size());
    for (auto* e : conds) {
        if (std::find(taken.begin(), taken.end(), e) != taken.end()) continue;
        std::vector<int> ts; expr_tuples(*e, ts);
        int di = -1;
        if (ts.size() == 1) for (size_t i = 0; i < out.dims.size(); i++) if (out.dims[i].tuple_id == ts[0]) di = (int)i;
        if (di >= 0) dim_conj[(size_t)di].push_back(e); else conj.push_back(e);
    }
    if (!lower_agg(in, out, agg, conj, fact, under_packet, false)) return false;
    out.kind = PK_STAR_AGG;
    Program dummy; memset(&dummy, 0, sizeof dummy);
    Lower lw{&out, &in, &dummy};
    for (size_t i = 0; i < out.dims.size(); i++) {
        StarDim& d = out.dims[i];
        d.key_col = lw.intern_col(d.tuple_id, d.key_col, in.slot_type(d.tuple_id, d.key_col));
        d.fk_col = lw.intern_col(fact, d.fk_col, in.slot_type(fact, d.fk_col));
        if (dim_conj[i].empty()) continue;
        d.n_filter = (int)dim_conj[i].size();
        if (!lower_own_program(in, out, d.filter, [&](Lower& l) { return l.predicate(dim_conj[i], 0, " on dimension " + std::to_string(d.tuple_id)); }))
            return false;
    }
    if ((int)out.cols.size() > MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
    for (size_t i = 0; i < out.cols.size(); i++) {
        out.col_side[i] = 0;
        for (size_t k = 0; k < out.dims.size(); k++) if (out.cols[i].tuple_id == out.dims[k].tuple_id) out.col_side[i] = 1 + (int)k;
    }
    // the aggregate runs over the gathered chunk
    std::string why; ColRef missing;
    const int r = lower_joined_row_agg(out, agg, conj, fact, under_packet, why, missing);
    if (r == 0) return in.fail(BKGPU_EUNSUPPORTED, "the aggregate over the joined row could not be lowered: %s", why.c_str());
    if (r < 0) return in.fail(BKGPU_EINVAL, "column %d_%d of the joined row is not a plan column", missing.tuple_id, missing.slot_id);
    return true;
}

// ---- APPLY: a correlated EXISTS / NOT EXISTS / [NOT] IN subquery under an aggregate ----
// [FILTER ->] APPLY(SEMI | ANTI_SEMI) with outer child [FILTER ->] SCAN and inner child (the subquery) [SORT ->] [FILTER ->]* SCAN.
// The reference's ApplyNode (src/exec/apply_node.cpp) runs an APPLY whose conditions hold no outer = inner column equality as a nested loop:
// for every outer row it puts the row's values in place of the outer columns inside the subquery and fetches the subquery's rows again
// (nested_loop_apply, replace_slot_ref_to_literal, fetcher_inner_table_data).  SEMI emits the outer row once if some subquery row makes
// every condition TRUE, ANTI_SEMI if none does (get_next_for_nested_loop_join); a NULL comparison is not TRUE.  Per outer row that is the
// SEMI / ANTI_SEMI join of the outer child with the subquery's scan, ON the APPLY's conditions and every subquery conjunct that reads the
// outer tuple (is_correlate_expr's classification), with the conjuncts that read the subquery alone as the inner child's own filter.  SEMI /
// ANTI_SEMI emit outer rows unchanged, so the filter between the aggregate and the APPLY, which reads the outer tuple alone, is part of the
// outer child's filter.  That JOIN is built here and lowered by lower_join_agg.
// An APPLY whose own conditions hold an outer = inner column equality (a correlated IN) runs as hash_apply instead: the subquery is opened
// once, with no outer row, so a correlated conjunct inside it reads the outer columns as NULL and no subquery row passes.  That is not the
// per-row meaning, and such a plan is refused.
//
// A scalar subquery: `x op (SELECT agg ... WHERE inner.k = outer.k ...)` reaches the library as APPLY(SEMI, max_one_row) whose subquery is
// AGG (no GROUP BY) -> [FILTER ->]* SCAN and whose conditions read the subquery's aggregates as AGG_EXPR nodes (construct_apply_node inlines the
// subquery's projections).  The reference runs it as nested_loop_apply: per outer row it substitutes the outer values into the subquery and
// runs it again.  A scalar AGG yields exactly one row even over no input — the default row of AggNode::get_next (agg_node.cpp:489-503), which
// needs a PACKET ancestor: get_parent_node walks up through the APPLY to the query's PACKET, and separate_apply leaves the subquery below the
// APPLY — so the row exists, with COUNT / COUNT(*) 0 and SUM / AVG / MIN / MAX NULL.  When every correlated conjunct is an outer = inner column
// equality, that per-row value is the group of the subquery's aggregate GROUP BY the inner columns (its own conjuncts as WHERE) whose key equals
// the outer values, or the empty-input row when there is none (a NULL outer key finds none; the NULL-key group is never found).  So the
// subquery becomes a grouped aggregate of its own (Compiled::sub), and the plan's aggregate runs over the outer rows plus one looked-up column
// per subquery aggregate its conditions read (k_apply_lookup); its predicate is the outer filter, the filter above the APPLY and the conditions.
static bool lower_scalar_apply(Infer& in, Compiled& out, const HNode& agg, const HNode& apply, const HNode& sa, bool under_packet, const HNode* above) {
    auto below = [](const HNode* n) { return n->ch.empty() ? nullptr : skip_passthrough(&n->ch[0], nullptr); };
    const HNode* o = skip_passthrough(&apply.ch[0], nullptr);
    const HNode* ofilt = nullptr;
    if (is_filter(o)) { ofilt = o; o = below(o); }
    if (o && o->node_type == BK_JOIN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "an APPLY whose outer child is a join is outside the GPU path");
    if (!o || o->node_type != BK_SCAN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "the outer child of an APPLY must be [FILTER ->] SCAN");
    if (ofilt && ofilt->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a filter below an APPLY is order dependent: outside the GPU path");
    const int ot = o->tuple_id, at = sa.agg_tuple_id;
    if (!sa.group_exprs.empty())
        return in.fail(BKGPU_EUNSUPPORTED, "a GROUP BY inside a scalar subquery is outside the GPU path (the reference fails at run time when it yields more than one row)");
    if (sa.limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "a LIMIT inside the subquery of an APPLY is outside the GPU path");
    for (const HExpr& f : sa.agg_fns) {
        static const char* const taken[] = {"count_star", "count", "sum", "avg", "min", "max"};
        if (f.distinct || std::none_of(std::begin(taken), std::end(taken), [&](const char* n) { return f.name == n; }))
            return in.fail(BKGPU_EUNSUPPORTED, "aggregate %s%s in a scalar subquery is outside the GPU path (COUNT(*), COUNT, SUM, AVG, MIN and MAX are lowered)",
                           f.name.c_str(), f.distinct ? " DISTINCT" : "");
    }
    // the subquery's own conjuncts, and its correlated ones: each an outer = inner column equality
    std::vector<const HExpr*> own, moved;
    const HNode* i = below(&sa);
    for (; is_filter(i) && i->limit == -1; i = below(i))
        for (auto& e : i->conjuncts) {
            std::vector<int> ts; expr_tuples(e, ts);
            (std::find(ts.begin(), ts.end(), ot) != ts.end() ? moved : own).push_back(&e);
        }
    if (i && (i->node_type == BK_LIMIT_NODE || i->limit != -1)) return in.fail(BKGPU_EUNSUPPORTED, "a LIMIT inside the subquery of an APPLY is outside the GPU path");
    if (i && i->node_type == BK_JOIN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "a join inside the subquery of an APPLY is outside the GPU path");
    if (!i || i->node_type != BK_SCAN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "the subquery of a max_one_row APPLY must be AGG -> [FILTER ->]* SCAN");
    const int it = i->tuple_id;
    if (it == ot) return in.fail(BKGPU_EINVAL, "both children of an APPLY scan tuple %d", it);
    if (at == ot || at == it) return in.fail(BKGPU_EINVAL, "the subquery's aggregate tuple %d is also a scanned tuple", at);
    std::vector<const HExpr*> ikeys, okeys;
    for (const HExpr* e : moved) {
        const bool eq = slot_eq(*e) && ((e->ch[0].tuple_id == ot && e->ch[1].tuple_id == it) || (e->ch[0].tuple_id == it && e->ch[1].tuple_id == ot));
        if (!eq) return in.fail(BKGPU_EUNSUPPORTED, "a correlated conjunct of a scalar subquery that is not an outer = inner column equality runs as the reference's "
                                "nested loop: outside the GPU path");
        const bool inner_first = e->ch[0].tuple_id == it;
        ikeys.push_back(&e->ch[inner_first ? 0 : 1]); okeys.push_back(&e->ch[inner_first ? 1 : 0]);
    }
    if (ikeys.empty()) return in.fail(BKGPU_EUNSUPPORTED, "a scalar subquery without an outer = inner column equality is outside the GPU path");
    // 1. the subquery's aggregate, grouped by its inner key columns, each cast to the type the equality compares in
    HNode grouped = sa;
    for (size_t k = 0; k < ikeys.size(); k++) {
        int cast;
        if (!join_key_cast(in, ikeys[k]->col_type, okeys[k]->col_type, cast)) return false;
        HExpr g = *ikeys[k]; g.col_type = cast;
        grouped.group_exprs.push_back(g);
    }
    auto sub = std::make_shared<Compiled>();
    sub->tuples = out.tuples; sub->in_sets = out.in_sets;
    if (!lower_agg(in, *sub, grouped, own, it, false, true)) return false;
    if ((int)sub->cols.size() > MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
    // 2. the outer aggregate: its predicate reads the subquery's aggregates as columns of the aggregate tuple
    std::vector<HExpr> rewritten;
    std::function<bool(HExpr&)> resolve = [&](HExpr& e) -> bool {
        if ((e.node_type == BK_AGG_EXPR || e.node_type == BK_SLOT_REF) && e.tuple_id == at) {
            const int slot = e.node_type == BK_AGG_EXPR ? e.final_slot : e.slot_id;
            int k = -1;
            for (size_t x = 0; x < sa.agg_fns.size(); x++) if (sa.agg_fns[x].final_slot == slot) k = (int)x;
            if (k < 0) return in.fail(BKGPU_EINVAL, "the conditions of a scalar subquery read slot %d_%d, which its aggregate does not compute", at, slot);
            const int prim = sub->ap.agg[k].out_prim, st = in.slot_type(at, slot);
            if (st != BK_INVALID_TYPE && st != prim) return in.fail(BKGPU_EINVAL, "slot %d_%d is declared as type %d, its aggregate yields %d", at, slot, st, prim);
            HExpr r; r.node_type = BK_SLOT_REF; r.tuple_id = at; r.slot_id = slot; r.col_type = prim;
            e = r;
            return true;
        }
        if (e.node_type == BK_SLOT_REF && e.tuple_id != ot)
            return in.fail(BKGPU_EINVAL, "a condition of a scalar subquery reads tuple %d: only the outer tuple %d and the subquery's aggregates reach it", e.tuple_id, ot);
        if (e.node_type == BK_AGG_EXPR) return in.fail(BKGPU_EINVAL, "a condition of a scalar subquery reads an aggregate of tuple %d", e.tuple_id);
        for (auto& c : e.ch) if (!resolve(c)) return false;
        return true;
    };
    for (const HNode* n : {ofilt, above, &apply}) if (n) for (const HExpr& e : n->conjuncts) rewritten.push_back(e);
    for (HExpr& e : rewritten) if (!resolve(e)) return false;
    std::vector<const HExpr*> conj;
    for (const HExpr& e : rewritten) conj.push_back(&e);
    if (!lower_agg(in, out, agg, conj, ot, under_packet, true)) return false;
    Program dummy; memset(&dummy, 0, sizeof dummy);
    Lower lw{&out, &in, &dummy};
    for (const HExpr* k : okeys) out.sub_key_cols.push_back(lw.intern_col(ot, k->slot_id, in.slot_type(ot, k->slot_id)));
    if ((int)out.cols.size() > MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d columns referenced", MAX_COLS);
    for (size_t c = 0; c < out.cols.size(); c++) {
        if (out.cols[c].tuple_id != at) continue;
        for (size_t x = 0; x < sa.agg_fns.size(); x++)
            if (sa.agg_fns[x].final_slot == out.cols[c].slot_id) { out.sub_out_cols.push_back((int)c); out.sub_out_agg.push_back((int)x); }
    }
    out.sub = sub;
    return true;
}

static bool lower_apply_agg(Infer& in, Compiled& out, const HNode& agg, const HNode& apply, bool under_packet, const HNode* above) {
    const int jt = apply.join_type;
    if (jt == BK_LEFT_JOIN) return in.fail(BKGPU_EUNSUPPORTED, "a LEFT apply (a scalar subquery) is outside the GPU path");
    if (jt != BK_SEMI_JOIN && jt != BK_ANTI_SEMI_JOIN) return in.fail(BKGPU_EUNSUPPORTED, "an APPLY of join type %d is outside the GPU path (SEMI / ANTI_SEMI are lowered)", jt);
    if (apply.max_one_row) {
        const HNode* s = apply.ch.size() == 2 ? skip_passthrough(&apply.ch[1], nullptr) : nullptr;
        if (jt == BK_SEMI_JOIN && !apply.is_select_field && apply.compare_type == BK_CMP_NULL && s && s->node_type == BK_AGG_NODE)
            return lower_scalar_apply(in, out, agg, apply, *s, under_packet, above);
        return in.fail(BKGPU_EUNSUPPORTED, "an APPLY with max_one_row (a subquery that must return at most one row) is outside the GPU path");
    }
    if (apply.is_select_field) return in.fail(BKGPU_EUNSUPPORTED, "an APPLY of a subquery in the select list is outside the GPU path");
    if (apply.compare_type != BK_CMP_NULL) return in.fail(BKGPU_EUNSUPPORTED, "an APPLY with an ANY / ALL / SOME comparison (compare_type %d) is outside the GPU path", apply.compare_type);
    if (apply.ch.size() != 2) return in.fail(BKGPU_EINVAL, "APPLY node needs two children");
    auto below = [](const HNode* n) { return n->ch.empty() ? nullptr : skip_passthrough(&n->ch[0], nullptr); };
    const HNode* o = skip_passthrough(&apply.ch[0], nullptr);
    const HNode* ofilt = nullptr;
    if (is_filter(o)) { ofilt = o; o = below(o); }
    if (o && o->node_type == BK_JOIN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "an APPLY whose outer child is a join is outside the GPU path");
    if (!o || o->node_type != BK_SCAN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "the outer child of an APPLY must be [FILTER ->] SCAN");
    if (ofilt && ofilt->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a filter below an APPLY is order dependent: outside the GPU path");
    const int ot = o->tuple_id;
    // the subquery: a SORT does not change which rows exist; every filter's conjuncts are classified
    std::vector<const HExpr*> own, moved;
    const HNode* i = skip_passthrough(&apply.ch[1], nullptr);
    if (i && i->node_type == BK_SORT_NODE && i->limit == -1) i = below(i);
    for (; is_filter(i) && i->limit == -1; i = below(i))
        for (auto& e : i->conjuncts) {
            std::vector<int> ts; expr_tuples(e, ts);
            (std::find(ts.begin(), ts.end(), ot) != ts.end() ? moved : own).push_back(&e);
        }
    if (i && (i->node_type == BK_AGG_NODE || i->node_type == BK_MERGE_AGG_NODE))
        return in.fail(BKGPU_EUNSUPPORTED, "an aggregate inside the subquery of an APPLY is outside the GPU path");
    if (i && (i->node_type == BK_LIMIT_NODE || i->limit != -1)) return in.fail(BKGPU_EUNSUPPORTED, "a LIMIT inside the subquery of an APPLY is outside the GPU path");
    if (i && i->node_type == BK_JOIN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "a join inside the subquery of an APPLY is outside the GPU path");
    if (!i || i->node_type != BK_SCAN_NODE) return in.fail(BKGPU_EUNSUPPORTED, "the subquery of an APPLY must be [SORT ->] [FILTER ->]* SCAN");
    const int it = i->tuple_id;
    if (it == ot) return in.fail(BKGPU_EINVAL, "both children of an APPLY scan tuple %d", it);
    auto key_eq = [&](const HExpr& e) {
        return slot_eq(e) && ((e.ch[0].tuple_id == ot && e.ch[1].tuple_id == it) || (e.ch[0].tuple_id == it && e.ch[1].tuple_id == ot));
    };
    if (std::any_of(apply.conjuncts.begin(), apply.conjuncts.end(), key_eq) && !moved.empty())
        return in.fail(BKGPU_EUNSUPPORTED, "a correlated IN subquery: the reference runs an APPLY whose conditions hold an outer = inner equality as hash_apply, "
                       "which reads the outer columns of the subquery's %zu correlated conjuncts as NULL instead of per outer row: outside the GPU path", moved.size());
    std::vector<const HExpr*> folded;
    if (above)
        for (auto& e : above->conjuncts) {
            std::vector<int> ts; expr_tuples(e, ts);
            for (int t : ts) if (t != ot) return in.fail(BKGPU_EINVAL, "the filter above an APPLY reads tuple %d: only the outer tuple %d reaches it", t, ot);
            folded.push_back(&e);
        }
    std::vector<const HExpr*> conds = conjuncts_of(&apply);
    conds.insert(conds.end(), moved.begin(), moved.end());
    if (std::none_of(conds.begin(), conds.end(), [&](const HExpr* e) { return key_eq(*e); }))
        return in.fail(BKGPU_EUNSUPPORTED, "an APPLY without an outer = inner column equality among its conditions and correlated conjuncts runs as the "
                       "reference's nested loop: outside the GPU path");
    // the decorrelated join: JOIN(outer [FILTER: own + folded] -> SCAN, inner [FILTER: own] -> SCAN) ON conditions + moved
    auto child = [](const HNode& scan, std::vector<const HExpr*> conj) {
        if (conj.empty()) return scan;
        HNode f; f.node_type = BK_WHERE_FILTER_NODE;
        for (auto* e : conj) f.conjuncts.push_back(*e);
        f.ch.push_back(scan);
        return f;
    };
    std::vector<const HExpr*> oconj = conjuncts_of(ofilt);
    oconj.insert(oconj.end(), folded.begin(), folded.end());
    HNode join; join.node_type = BK_JOIN_NODE; join.join_type = jt; join.limit = apply.limit;
    for (auto* e : conds) join.conjuncts.push_back(*e);
    join.ch.push_back(child(*o, oconj));
    join.ch.push_back(child(*i, own));
    if (!lower_join_agg(in, out, agg, join, under_packet, nullptr)) return false;
    out.apply_join_type = jt; out.apply_moved = (int)moved.size(); out.apply_folded = (int)folded.size();
    return true;
}

// A JOIN whose rows are the result ([LIMIT ->] [SORT ->] [FILTER ->] JOIN; JoinNode::get_next, join_node.cpp:1200-1326).  The joined rows that
// pass the conditions are produced on the device batch by batch (pairs + one gather per column) and handed to a sink fragment
// (Compiled::post, kind PK_FILTER without a predicate, or PK_SORT) whose "scan tuple" is the joined row: every slot of both tuples.
// INNER: child filters, the residual conditions and a filter above the join are one predicate.  LEFT / RIGHT: the outer (build) side is
// preserved, unmatched rows come out NULL-extended; the inner child's filter is its own program (as in lower_join_agg), a filter on the
// preserved child or above the join is refused.  FULL: both sides
// are preserved; a filter above the join is the sink's predicate, so it also judges the NULL-extended rows.
static bool lower_join_rows(Infer& in, Compiled& out, const HNode& join, const HNode* above, const HNode* sort, const HNode* limit_node) {
    int jt = join.join_type;
    if (jt != BK_INNER_JOIN && jt != BK_LEFT_JOIN && jt != BK_RIGHT_JOIN && jt != BK_FULL_JOIN)
        return in.fail(BKGPU_EUNSUPPORTED, "a join of type %d that returns rows is outside the GPU path (INNER / LEFT / RIGHT / FULL are lowered)", jt);
    if (join.ch.size() != 2) return in.fail(BKGPU_EINVAL, "JOIN node needs two children");
    if (above && above->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a filter above a join: use a LIMIT node");
    const HNode *side[2], *filt[2];
    if (!join_children(in, join, jt, side, filt)) return false;
    const bool full = jt == BK_FULL_JOIN;
    if (full && (filt[0] || filt[1])) return in.fail(BKGPU_EUNSUPPORTED, "FULL join over filtered children is outside the GPU path");
    if (jt == BK_LEFT_JOIN && above) return in.fail(BKGPU_EUNSUPPORTED, "LEFT join with a filter above it is outside the GPU path");
    if (jt == BK_LEFT_JOIN && filt[0]) return in.fail(BKGPU_EUNSUPPORTED, "a filter on the preserved side of a LEFT / RIGHT join is outside the GPU path");
    const int build_tuple = side[0]->tuple_id, probe_tuple = side[1]->tuple_id;
    out.kind = PK_JOIN; out.build_tuple = build_tuple; out.scan_tuple = probe_tuple; out.join_type = jt;
    std::vector<const HExpr*> conj;
    const HExpr *bk, *pk;
    if (!join_equality(in, join, build_tuple, probe_tuple, bk, pk, conj)) return false;
    if (jt == BK_INNER_JOIN) for (int i = 0; i < 2; i++) if (filt[i]) for (auto& e : filt[i]->conjuncts) conj.push_back(&e);
    if (above && !full) for (auto& e : above->conjuncts) conj.push_back(&e);   // (FULL: the sink's predicate, below)
    if (!join_key_cast(in, bk->col_type, pk->col_type, out.join_key_prim)) return false;
    Program& p = out.prog; memset(&p, 0, sizeof p);
    memset(&out.ap, 0, sizeof out.ap);
    Lower lw{&out, &in, &p};
    // every slot of both tuples is an output column (and a device column): build tuple first, as the joined row lists them
    if (!intern_tuple(in, out, lw, build_tuple, "join tuple", "the joined row") || !intern_tuple(in, out, lw, probe_tuple, "join tuple", "the joined row")) return false;
    const size_t n_payload = out.cols.size();
    out.build_key_col = lw.intern_col(bk->tuple_id, bk->slot_id, in.slot_type(bk->tuple_id, bk->slot_id));
    out.probe_key_col = lw.intern_col(pk->tuple_id, pk->slot_id, in.slot_type(pk->tuple_id, pk->slot_id));
    int reg = 0;
    out.ap.pred_out = -1;
    if (!conj.empty()) {
        out.ap.pred_out = reg;
        if (!lw.predicate(conj, reg++)) return false;
    }
    p.n_out = reg;
    if (jt == BK_LEFT_JOIN && !lower_child_filter(in, out, filt[1], probe_tuple, out.probe_filter, out.n_probe_filter)) return false;
    if (out.cols.size() != n_payload) return in.fail(BKGPU_EINVAL, "join conditions reference a slot that is in neither tuple descriptor");
    // the sink over the joined rows.  FULL: the filter above the join judges every joined row, the NULL-extended ones included, after the
    // match decision
    if (!lower_sink(in, out, {sort, full ? above : nullptr, join.limit, false, "columns in the joined row under a sink",
                              "ORDER BY above a join references a column outside the joined row"}, limit_node)) return false;
    out.limit = out.post->limit; out.offset = out.post->offset;
    return true;
}

// ---------------------------------------------------------------- window
// [LIMIT ->] [SORT ->] (WINDOW -> SORT){1..8} [FILTER ->] SCAN (select_planner.cpp:705-760): the planner gives every window spec its own
// SORT by the partition expressions followed by the order expressions (is_null_first = is_asc) and a WINDOW that keeps the order part.
// Each pair becomes one stage over the retained scan rows; the operators above the top WINDOW are the query's ORDER BY / LIMIT.
namespace {
struct WinName { const char* name; int kind; };
const WinName k_win_names[] = {{"count_star", WF_COUNT_STAR}, {"count", WF_COUNT}, {"sum", WF_SUM}, {"avg", WF_AVG}, {"min", WF_MIN}, {"max", WF_MAX},
                               {"row_number", WF_ROW_NUMBER}, {"rank", WF_RANK}, {"dense_rank", WF_DENSE_RANK}, {"percent_rank", WF_PERCENT_RANK},
                               {"cume_dist", WF_CUME_DIST}, {"ntile", WF_NTILE}, {"lead", WF_LEAD}, {"lag", WF_LAG}, {"first_value", WF_FIRST_VALUE},
                               {"last_value", WF_LAST_VALUE}, {"nth_value", WF_NTH_VALUE}};
bool win_is_agg(int k) { return k <= WF_MAX; }
bool win_no_frame(int k) { return k >= WF_ROW_NUMBER && k <= WF_LAG; }
// the value of an INT_LITERAL argument; false when the node is not one
bool int_literal(const HExpr& e, int64_t& v) {
    if (e.node_type != BK_INT_LITERAL || e.lit_null) return false;
    v = (int64_t)e.lit_bits;
    return true;
}
std::string sort_key_text(const HNode& s) {
    std::string k;
    for (size_t i = 0; i < s.order_exprs.size(); i++) k += expr_key(s.order_exprs[i]) + (s.is_asc[i] ? "A" : "D") + (s.is_null_first[i] ? "F" : "L");
    return k;
}
}  // namespace

// (MERGE_)AGG -> [FILTER ->] SCAN / JOIN / APPLY: the aggregate, lowered into `out` (the aggregate root of a fragment, or the aggregate below
// window stages)
static bool lower_agg_node(Infer& in, Compiled& out, const HNode& top, bool under_packet) {
    if (top.ch.empty()) return in.fail(BKGPU_EINVAL, "AGG node without a child");
    const HNode* c = skip_passthrough(&top.ch[0], nullptr);
    const HNode* filter = nullptr;
    if (is_filter(c)) { filter = c; c = c->ch.empty() ? nullptr : skip_passthrough(&c->ch[0], nullptr); }
    if (!c || (c->node_type != BK_SCAN_NODE && c->node_type != BK_JOIN_NODE && c->node_type != BK_APPLY_NODE)) return in.fail(BKGPU_EUNSUPPORTED, "AGG child must be [FILTER ->] SCAN or JOIN");
    if (filter && filter->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a filter below an aggregate is order dependent: outside the GPU path");
    bool ok;
    if (c->node_type == BK_SCAN_NODE) ok = lower_agg(in, out, top, conjuncts_of(filter), c->tuple_id, under_packet, true);
    else if (c->node_type == BK_APPLY_NODE) ok = lower_apply_agg(in, out, top, *c, under_packet, filter);
    // AGG -> [FILTER ->] JOIN: the store-side chain of a filtered join (separate.cpp:241-260)
    else ok = join_leaves(c) > 2 ? lower_star_agg(in, out, top, *c, under_packet, filter) : lower_join_agg(in, out, top, *c, under_packet, filter);
    if (!ok) return false;
    bool hll_out = false, hll_merge = false, rb_out = false;
    for (const OutCol& oc : out.out_cols) { hll_out = hll_out || oc.kind == 2; rb_out = rb_out || oc.kind == 3; }
    for (int k = 0; k < out.ap.n_agg; k++) hll_merge = hll_merge || (out.ap.agg[k].kind == AG_HLL && out.ap.agg[k].arg_prim == BK_HLL);
    if (hll_merge && out.kind != PK_AGG)   // (a join would have to gather 16400-byte values to the probe rows)
        return in.fail(BKGPU_EUNSUPPORTED, "MERGE_AGG of HLL sketches over a join is outside the GPU path (MERGE_AGG over a scan is lowered)");
    if (rb_out && out.ap.n_hll) return in.fail(BKGPU_EUNSUPPORTED, "rb_build_agg beside hll_add_agg in one aggregate is outside the GPU path");
    return true;
}

// The WINDOW -> SORT pairs of `w` (a PK_WINDOW fragment whose input columns are interned already), bottom-up, then the window output columns
// and the query's ORDER BY [+ LIMIT / OFFSET] above them.  `outside`: the refusal of a window expression that reads a column the input
// rows do not hold.
using WinPairs = std::vector<std::pair<const HNode*, const HNode*>>;   // (WINDOW, SORT), top-down
static bool lower_win_stages(Infer& in, Compiled& out, const WinPairs& pairs, const HNode* outer_sort, const HNode* limit_node, const std::string& outside) {
    const size_t n_scan_cols = out.cols.size();
    // one device program per distinct (expression, result type) of a stage
    auto intern_expr = [&](WinStage& st, std::map<std::string, int>& seen, const HExpr& e, int to) -> int {
        const std::string key = expr_key(e) + ":" + std::to_string(to);
        auto it = seen.find(key);
        if (it != seen.end()) return it->second;
        Program q;
        if (!lower_own_program(in, out, q, [&](Lower& l) { int depth = 0; return l.expr(e, depth) && l.cast(e.col_type, to) && l.out_reg(0); })) return -1;
        if (out.cols.size() != n_scan_cols) { in.fail(BKGPU_EUNSUPPORTED, "%s", outside.c_str()); return -1; }
        st.exprs.push_back(q); st.expr_prim.push_back(to);
        return seen[key] = (int)st.exprs.size() - 1;
    };
    std::string prev_keys;
    size_t n_fns = 0, n_sorts = 0;
    std::vector<OutCol> win_cols;
    for (size_t pi = pairs.size(); pi-- > 0;) {   // bottom-up: the order the rows pass through them
        const HNode& W = *pairs[pi].first;
        const HNode& S = *pairs[pi].second;
        WinStage st;
        std::map<std::string, int> seen;
        if (W.limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "a LIMIT on a WINDOW node (the subquery rewrite's) is outside the GPU path");
        if (S.limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "a LIMIT on a window's SORT node is outside the GPU path");
        const size_t np = W.group_exprs.size(), no = W.order_exprs.size();
        bool match = S.order_exprs.size() == np + no;
        for (size_t k = 0; match && k < S.order_exprs.size(); k++) {
            const HExpr& want = k < np ? W.group_exprs[k] : W.order_exprs[k - np];
            match = expr_key(want) == expr_key(S.order_exprs[k]) && S.is_null_first[k] == S.is_asc[k] && (k < np || (S.is_asc[k] != 0) == (W.is_asc[k - np] != 0));
        }
        if (!match) return in.fail(BKGPU_EUNSUPPORTED, "the SORT below a WINDOW must order by its partition expressions, then its order expressions");
        if (np + no > 4) return in.fail(BKGPU_EUNSUPPORTED, "more than 4 partition and order expressions in one window");
        for (size_t k = 0; k < np; k++) {
            const int ct = W.group_exprs[k].col_type;
            if (ct == BK_STRING) return in.fail(BKGPU_EUNSUPPORTED, "PARTITION BY over a STRING key is outside the GPU path");
            if (is_double_t(ct)) return in.fail(BKGPU_EUNSUPPORTED, "PARTITION BY over a FLOAT / DOUBLE key is outside the GPU path: its byte encoding separates values the sort treats as equal");
        }
        for (size_t k = 0; k < no; k++)
            if (W.order_exprs[k].col_type == BK_STRING) return in.fail(BKGPU_EUNSUPPORTED, "window ORDER BY over a STRING key is outside the GPU path");
        for (size_t k = 0; k < S.order_exprs.size(); k++) {
            const HExpr& e = S.order_exprs[k];
            const int x = intern_expr(st, seen, e, e.col_type);
            if (x < 0) return false;
            st.sort_keys.push_back({x, e.col_type, S.is_asc[k] != 0, S.is_null_first[k] != 0});
        }
        st.n_part = (int)np;
        const std::string keys = sort_key_text(S);
        st.new_sort = !S.order_exprs.empty() && keys != prev_keys;   // (no keys: OVER () keeps the current order; equal keys: a stable re-sort is the identity)
        if (!S.order_exprs.empty()) prev_keys = keys;
        if (st.new_sort && ++n_sorts > 8) return in.fail(BKGPU_EUNSUPPORTED, "more than 8 distinct window sorts in one fragment");
        // frame (WindowProcessor::init, window_node.cpp:337-394; Row/RangeFrameWindowProcessor::get_start_row / get_end_row)
        st.has_frame = W.has_frame;
        st.frame_type = W.frame_type;
        if (W.has_frame) {
            if (W.frame_type != BK_FRAME_ROWS && W.frame_type != BK_FRAME_RANGE) return in.fail(BKGPU_EINVAL, "bad window frame type %d", W.frame_type);
            const HFrameBound* hb[2] = {&W.frame_start, &W.frame_end};
            WinBound* wb[2] = {&st.start, &st.end};
            for (int b = 0; b < 2; b++) {
                const HFrameBound& h = *hb[b];
                if (h.type < BK_BT_PRECEDING || h.type > BK_BT_CURRENT_ROW) return in.fail(BKGPU_EINVAL, "bad window frame bound type %d", h.type);
                if (h.unbounded && b == 0 && h.type != BK_BT_PRECEDING) return in.fail(BKGPU_EUNSUPPORTED, "an unbounded frame start must be UNBOUNDED PRECEDING");
                if (h.unbounded && b == 1 && h.type != BK_BT_FOLLOWING) return in.fail(BKGPU_EUNSUPPORTED, "an unbounded frame end must be UNBOUNDED FOLLOWING");
                wb[b]->type = h.type; wb[b]->unbounded = h.unbounded; wb[b]->num = 0;
                if (!h.unbounded && h.type != BK_BT_CURRENT_ROW) {
                    int64_t v = -1;
                    if (!h.has_expr || !int_literal(h.expr, v) || v < 0 || v > INT32_MAX) return in.fail(BKGPU_EUNSUPPORTED, "a window frame offset must be an integer literal >= 0");
                    if (W.frame_type == BK_FRAME_RANGE) return in.fail(BKGPU_EUNSUPPORTED, "a RANGE frame with an offset is outside the GPU path (the reference fails at run time)");
                    wb[b]->num = v;
                }
            }
            if (W.frame_type == BK_FRAME_ROWS && !st.start.unbounded && !st.end.unbounded) {
                auto pos = [](const WinBound& x) { return x.type == BK_BT_PRECEDING ? -x.num : (x.type == BK_BT_FOLLOWING ? x.num : 0); };
                if (pos(st.end) - pos(st.start) + 1 > 4096) return in.fail(BKGPU_EUNSUPPORTED, "a bounded ROWS frame wider than 4096 rows is outside the GPU path");
            }
        }
        const bool whole = !st.has_frame || (st.start.unbounded && st.end.unbounded);
        int method = WM_FWD;
        if (!whole) {
            if (st.start.unbounded) method = WM_FWD;
            else if (st.end.unbounded) method = WM_BWD;
            else if (st.frame_type == BK_FRAME_RANGE) method = WM_PEER;
            else method = WM_DIRECT;
        }
        for (const HExpr& f : W.agg_fns) {
            if (f.node_type != BK_WINDOW_EXPR) return in.fail(BKGPU_EINVAL, "a WINDOW node's function must be a WINDOW_EXPR");
            WinFn wf;
            wf.kind = -1;
            for (const WinName& nm : k_win_names) if (f.name == nm.name) wf.kind = nm.kind;
            if (wf.kind < 0) return in.fail(BKGPU_EUNSUPPORTED, "window function '%s' is outside the GPU path", f.name.c_str());
            wf.tuple_id = f.tuple_id; wf.slot_id = f.slot_id; wf.out_prim = f.col_type;
            if (st.has_frame && win_no_frame(wf.kind)) return in.fail(BKGPU_EUNSUPPORTED, "a frame on %s() is outside the GPU path (the planner never emits one)", f.name.c_str());
            const bool takes_value = wf.kind != WF_COUNT_STAR && wf.kind != WF_ROW_NUMBER && wf.kind != WF_RANK && wf.kind != WF_DENSE_RANK &&
                                     wf.kind != WF_PERCENT_RANK && wf.kind != WF_CUME_DIST && wf.kind != WF_NTILE;
            if (takes_value) {
                if (f.ch.empty()) return in.fail(BKGPU_EINVAL, "window %s() without an argument", f.name.c_str());
                const HExpr& x = f.ch[0];
                if (x.col_type == BK_STRING) return in.fail(BKGPU_EUNSUPPORTED, "window %s() over a STRING argument is outside the GPU path", f.name.c_str());
                if ((wf.kind == WF_SUM || wf.kind == WF_AVG) && is_datetime_family(x.col_type))
                    return in.fail(BKGPU_EUNSUPPORTED, "window %s() over a date/time argument is outside the GPU path", f.name.c_str());
                // SUM / AVG read value.cast_to(_col_type); MIN / MAX / LEAD / LAG / FIRST / LAST / NTH keep the argument's type
                wf.arg_prim = wf.kind == WF_COUNT ? x.col_type : wf.out_prim;
                if ((wf.arg = intern_expr(st, seen, x, wf.arg_prim)) < 0) return false;
            }
            if (wf.kind == WF_NTILE && (f.ch.empty() || !int_literal(f.ch[0], wf.n) || wf.n <= 0)) return in.fail(BKGPU_EUNSUPPORTED, "NTILE needs an integer literal > 0");
            if (wf.kind == WF_NTH_VALUE && (f.ch.size() < 2 || !int_literal(f.ch[1], wf.n) || wf.n <= 0)) return in.fail(BKGPU_EUNSUPPORTED, "NTH_VALUE needs an integer literal > 0");
            if (wf.kind == WF_NTH_VALUE && wf.n > INT32_MAX)   // (the reference reads row start + n - 1 through an int: no meaning past it)
                return in.fail(BKGPU_EUNSUPPORTED, "NTH_VALUE with n > 2147483647 is outside the GPU path (the reference truncates the row index to int)");
            if (wf.kind == WF_LEAD || wf.kind == WF_LAG) {
                wf.n = 1;
                if (f.ch.size() > 1 && (!int_literal(f.ch[1], wf.n) || wf.n < 0)) return in.fail(BKGPU_EUNSUPPORTED, "the LEAD / LAG offset must be an integer literal >= 0");
                if (f.ch.size() > 2) {
                    if (f.ch[2].col_type == BK_STRING) return in.fail(BKGPU_EUNSUPPORTED, "a STRING LEAD / LAG default is outside the GPU path");
                    if ((wf.def = intern_expr(st, seen, f.ch[2], wf.out_prim)) < 0) return false;   // default_expr->get_value(current row).cast_to(_col_type)
                }
            }
            wf.method = win_is_agg(wf.kind) ? method : WM_NONE;
            st.fns.push_back(wf);
            win_cols.push_back({wf.tuple_id, wf.slot_id, wf.out_prim, 0});
            if (++n_fns > 32) return in.fail(BKGPU_EUNSUPPORTED, "more than 32 window functions in one fragment");
        }
        out.win.push_back(std::move(st));
    }
    for (const OutCol& oc : win_cols) {
        for (const OutCol& x : out.out_cols)
            if (x.tuple_id == oc.tuple_id && x.slot_id == oc.slot_id) return in.fail(BKGPU_EINVAL, "window output column %d_%d appears twice", oc.tuple_id, oc.slot_id);
        out.out_cols.push_back(oc);
    }
    out.limit = -1; out.offset = 0;
    if (outer_sort)   // the query's ORDER BY over the window rows (window columns included) [+ LIMIT / OFFSET]
        return lower_sink(in, out, {outer_sort, nullptr, -1, true, "window output columns under an ORDER BY",
                                    "SORT / HAVING above an aggregate references a column the aggregate does not output"}, limit_node);
    merge_limit(limit_node, out.limit, out.offset);   // LIMIT / OFFSET over the top stage's order
    return true;
}

// [LIMIT ->] [SORT ->] (WINDOW -> SORT){1..8} [HAVING ->] (MERGE_)AGG (select_planner.cpp:147-171): the aggregate is lowered as it is without
// the windows; the stages become its post fragment (kind PK_WINDOW) over the aggregate's output rows, HAVING that fragment's predicate.
// The windows sit above the db-side aggregate only: a MERGE_AGG over the stores' partial rows (separate.cpp:241-259), or an aggregate over a
// join / APPLY.  An AGG straight over a scan is the store-side aggregate, which the planner never puts under a window.
static bool lower_window_over_agg(Infer& in, Compiled& out, const WinPairs& pairs, const HNode* having, const HNode& agg, const HNode* outer_sort,
                                  const HNode* limit_node, bool under_packet) {
    if (having && having->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a HAVING filter below a window is order dependent");
    if (!lower_agg_node(in, out, agg, under_packet)) return false;
    for (const OutCol& oc : out.out_cols) {
        if (oc.kind == 3) return in.fail(BKGPU_EUNSUPPORTED, "a window above an aggregate that returns a BITMAP is outside the GPU path");
        if (oc.kind == 2) return in.fail(BKGPU_EUNSUPPORTED, "a window above an aggregate that returns an HLL sketch is outside the GPU path");
    }
    if (out.out_cols.size() > (size_t)MAX_COLS) return in.fail(BKGPU_EUNSUPPORTED, "more than %d aggregate output columns under a window", MAX_COLS);
    auto post = std::make_shared<Compiled>();
    Compiled& w = *post;
    w.kind = PK_WINDOW;
    w.tuples = out.tuples; w.scan_tuple = -1; w.in_sets = out.in_sets;
    Program& p = w.prog; memset(&p, 0, sizeof p);
    memset(&w.ap, 0, sizeof w.ap);
    Lower lw{&w, &in, &p};
    // the input row: the aggregate's output columns in order (AVG's intermediate blob rides along as a 16-byte payload column)
    for (const OutCol& oc : out.out_cols) {
        if (lw.intern_col(oc.tuple_id, oc.slot_id, oc.prim) != (int)w.out_cols.size())
            return in.fail(BKGPU_EUNSUPPORTED, "aggregate output columns %d_%d appear twice", oc.tuple_id, oc.slot_id);
        w.out_cols.push_back(oc);
    }
    int reg = 0;
    if (!lower_predicate(lw, having, w.ap, reg)) return false;
    p.n_out = reg;
    if (w.cols.size() != out.out_cols.size()) return in.fail(BKGPU_EUNSUPPORTED, "HAVING below a window references a column the aggregate does not output");
    if (!lower_win_stages(in, w, pairs, outer_sort, limit_node, "a window expression reads a column the aggregate does not output")) return false;
    out.post = post;
    return true;
}

// [LIMIT ->] [SORT ->] (WINDOW -> SORT){1..8} [FILTER ->] SCAN (select_planner.cpp:705-760): the planner gives every window spec its own
// SORT by the partition expressions followed by the order expressions (is_null_first = is_asc) and a WINDOW that keeps the order part.
// Each pair becomes one stage over the retained scan rows; the operators above the top WINDOW are the query's ORDER BY / LIMIT.  Above an
// aggregate: lower_window_over_agg.
static bool lower_window(Infer& in, Compiled& out, const HNode& wtop, const HNode* outer_sort, const HNode* limit_node, bool under_packet) {
    WinPairs pairs;
    const HNode* t = &wtop;
    while (t && t->node_type == BK_WINDOW_NODE) {
        const HNode* s = t->ch.empty() ? nullptr : skip_passthrough(&t->ch[0], nullptr);
        if (!s || s->node_type != BK_SORT_NODE || s->ch.empty()) return in.fail(BKGPU_EUNSUPPORTED, "a WINDOW node's child must be its SORT node");
        pairs.push_back({t, s});
        t = skip_passthrough(&s->ch[0], nullptr);
    }
    {   // [HAVING ->] (MERGE_)AGG over the stores' rows, a join or an APPLY
        const HNode* having = nullptr;
        const HNode* a = t;
        if (a && (is_filter(a) || a->node_type == BK_HAVING_FILTER_NODE)) { having = a; a = a->ch.empty() ? nullptr : skip_passthrough(&a->ch[0], nullptr); }
        if (a && (a->node_type == BK_AGG_NODE || a->node_type == BK_MERGE_AGG_NODE) && !a->ch.empty()) {
            const HNode* src = skip_passthrough(&a->ch[0], nullptr);
            if (is_filter(src)) src = src->ch.empty() ? nullptr : skip_passthrough(&src->ch[0], nullptr);
            const bool over_scan = src && src->node_type == BK_SCAN_NODE;
            const bool over_rows = src && (src->node_type == BK_JOIN_NODE || src->node_type == BK_APPLY_NODE);
            if ((over_scan && a->node_type == BK_MERGE_AGG_NODE) || over_rows)
                return lower_window_over_agg(in, out, pairs, having, *a, outer_sort, limit_node, under_packet);
        }
    }
    out.kind = PK_WINDOW;
    const HNode* filter = nullptr;
    if (is_filter(t)) { filter = t; t = t->ch.empty() ? nullptr : skip_passthrough(&t->ch[0], nullptr); }
    if (!t || t->node_type != BK_SCAN_NODE)
        return in.fail(BKGPU_EUNSUPPORTED, "window stages must sit on [FILTER ->] SCAN: a window over an aggregate or a join is outside the GPU path");
    if (filter && filter->limit != -1) return in.fail(BKGPU_EUNSUPPORTED, "LIMIT on a filter below a window is order dependent");
    out.scan_tuple = t->tuple_id;
    Program& p = out.prog; memset(&p, 0, sizeof p);
    memset(&out.ap, 0, sizeof out.ap);
    Lower lw{&out, &in, &p};
    if (!intern_tuple(in, out, lw, t->tuple_id, "scan tuple", "the scan tuple")) return false;
    int reg = 0;
    if (!lower_predicate(lw, filter, out.ap, reg)) return false;
    p.n_out = reg;
    return lower_win_stages(in, out, pairs, outer_sort, limit_node, "a window expression reads a column outside the scan tuple " + std::to_string(out.scan_tuple));
}

// ---------------------------------------------------------------- entry
// [SORT ->] [FILTER ->] JOIN / APPLY (`node_type`) at the top of the fragment -> that node, else nullptr
static const HNode* rows_shape(const HNode* t, int node_type) {
    if (t && t->node_type == BK_SORT_NODE && !t->ch.empty()) t = skip_passthrough(&t->ch[0], nullptr);
    if (t && is_filter(t) && !t->ch.empty()) t = skip_passthrough(&t->ch[0], nullptr);
    return t && t->node_type == node_type ? t : nullptr;
}

int compile_plan(const uint8_t* desc, size_t len, Compiled& out, std::string& err) {
    if (!desc || len < 16 || (len & 3)) { err = "plan descriptor is empty or not a multiple of 4 bytes"; return BKGPU_EINVAL; }
    Reader r{}; r.w = (const int32_t*)desc; r.n = len / 4;
    if ((uint32_t)r.rd() != BKGPU_PLAN_MAGIC) { err = "bad plan magic"; return BKGPU_EINVAL; }
    if (r.rd() != BKGPU_PLAN_VERSION) { err = "unsupported plan version"; return BKGPU_EINVAL; }
    int nt = r.rd(), nn = r.rd();
    if (nt < 0 || nt > 16 || nn <= 0 || nn > 64) { err = "bad tuple / node count"; return BKGPU_EINVAL; }
    for (int i = 0; i < nt && !r.fail; i++) {
        HTuple t; t.tuple_id = r.rd(); int ns = r.rd();
        if (ns < 0 || ns > 4096) { r.bad("bad slot count"); break; }
        for (int k = 0; k < ns; k++) { int sid = r.rd(); int pt = r.rd(); t.slots.push_back({sid, pt}); }
        out.tuples.push_back(t);
    }
    HNode root;
    if (!r.fail) parse_node(r, root, nn, 0);
    if (!r.fail && nn != 0) r.bad("plan node count mismatch");
    if (!r.fail && r.pos != r.n) r.bad("trailing words after the plan");
    if (r.fail) { err = r.err; return r.err.find("outside the GPU path") != std::string::npos ? BKGPU_EUNSUPPORTED : BKGPU_EINVAL; }
    Infer in{}; in.tuples = &out.tuples;
    if (!infer_node(in, root)) { err = in.err; return in.code; }
    out.in_sets = std::make_shared<InSets>();

    bool under_packet = false;
    const HNode* top = skip_passthrough(&root, &under_packet);
    if (!top) { err = "empty plan"; return BKGPU_EINVAL; }
    bool ok = false;
    const HNode* limit_node = nullptr;
    if (top->node_type == BK_LIMIT_NODE && !top->ch.empty()) { limit_node = top; top = skip_passthrough(&top->ch[0], &under_packet); }
    // the db-side chain above an aggregate: [LIMIT ->] [SORT ->] [HAVING_FILTER ->] (MERGE_)AGG (separate.cpp:241-260): the operators
    // above the aggregate become a post fragment over the aggregate's output rows
    const HNode *post_sort = nullptr, *post_having = nullptr;
    {
        const HNode* t = top;
        const HNode *ps = nullptr, *ph = nullptr;
        if (t->node_type == BK_SORT_NODE && !t->ch.empty()) { ps = t; t = skip_passthrough(&t->ch[0], nullptr); }
        if (t && (is_filter(t) || t->node_type == BK_HAVING_FILTER_NODE) && !t->ch.empty()) { ph = t; t = skip_passthrough(&t->ch[0], nullptr); }
        if (t && (ps || ph) && (t->node_type == BK_AGG_NODE || t->node_type == BK_MERGE_AGG_NODE)) { post_sort = ps; post_having = ph; top = t; }
    }
    const HNode* win_sort = nullptr;   // [SORT ->] WINDOW: the query's ORDER BY above the window stages
    if (top->node_type == BK_SORT_NODE && !top->ch.empty()) {
        const HNode* c = skip_passthrough(&top->ch[0], nullptr);
        if (c && c->node_type == BK_WINDOW_NODE) win_sort = top;
    }
    if (win_sort || top->node_type == BK_WINDOW_NODE) {
        ok = lower_window(in, out, win_sort ? *skip_passthrough(&win_sort->ch[0], nullptr) : *top, win_sort, limit_node, under_packet);
    } else if (top->node_type == BK_AGG_NODE || top->node_type == BK_MERGE_AGG_NODE) {
        ok = lower_agg_node(in, out, *top, under_packet);
        // LimitNode straight over the aggregate: the result extraction (agg_result) skips `offset` groups and then keeps `limit` of them,
        // so the limit is stored as it is — not as the first limit + offset rows that a sort or a filter keeps before skipping
        if (ok && limit_node && !post_sort && !post_having) { out.limit = limit_node->limit; out.offset = limit_node->offset; }
        bool hll_out = false, rb_out = false;
        for (const OutCol& oc : out.out_cols) { hll_out = hll_out || oc.kind == 2; rb_out = rb_out || oc.kind == 3; }
        if (ok && (post_sort || post_having) && rb_out) {
            err = "a SORT / HAVING / LIMIT above an aggregate that returns a BITMAP is outside the GPU path"; return BKGPU_EUNSUPPORTED;
        }
        if (ok && (post_sort || post_having) && hll_out) {
            err = "a SORT / HAVING / LIMIT above an aggregate that returns an HLL sketch is outside the GPU path"; return BKGPU_EUNSUPPORTED;
        }
        if (ok && (post_sort || post_having))
            ok = lower_sink(in, out, {post_sort, post_having, post_having ? post_having->limit : -1, true, "aggregate output columns under a SORT / HAVING",
                                      "SORT / HAVING above an aggregate references a column the aggregate does not output"}, limit_node);
    } else if (rows_shape(top, BK_APPLY_NODE)) {
        err = "an APPLY (correlated subquery) that returns rows is outside the GPU path (an aggregate over it is lowered)"; return BKGPU_EUNSUPPORTED;
    } else if (const HNode* jn = rows_shape(top, BK_JOIN_NODE)) {   // [SORT ->] [FILTER ->] JOIN: a join that returns its rows
        const HNode* t = top; const HNode *js = nullptr, *jf = nullptr;
        if (t->node_type == BK_SORT_NODE) { js = t; t = skip_passthrough(&t->ch[0], nullptr); }
        if (is_filter(t)) jf = t;
        if (join_leaves(jn) > 2) { err = "a join of more than two tables that returns rows is outside the GPU path (an aggregate over a star join is lowered)"; return BKGPU_EUNSUPPORTED; }
        ok = lower_join_rows(in, out, *jn, jf, js, limit_node);
    } else if (top->node_type == BK_SORT_NODE) {
        const HNode* c = top->ch.empty() ? nullptr : skip_passthrough(&top->ch[0], nullptr);
        const HNode* filter = nullptr;
        if (is_filter(c)) { filter = c; c = c->ch.empty() ? nullptr : skip_passthrough(&c->ch[0], nullptr); }
        if (!c || c->node_type != BK_SCAN_NODE) { err = "SORT child must be [FILTER ->] SCAN"; return BKGPU_EUNSUPPORTED; }
        ok = lower_sort(in, out, *top, filter, *c);
        if (ok) merge_limit(limit_node, out.limit, out.offset);
    } else if (is_filter(top) || top->node_type == BK_SCAN_NODE) {
        const HNode* c = top;
        if (is_filter(c)) c = c->ch.empty() ? nullptr : skip_passthrough(&c->ch[0], nullptr);
        if (!c || c->node_type != BK_SCAN_NODE) { err = "FILTER child must be SCAN"; return BKGPU_EUNSUPPORTED; }
        ok = lower_filter(in, out, limit_node, *top, *c);
    } else { err = "plan root is outside the GPU path"; return BKGPU_EUNSUPPORTED; }
    if (!ok) { err = in.err.empty() ? "plan could not be lowered" : in.err; return in.code ? in.code : BKGPU_EUNSUPPORTED; }
    explain(out);
    return BKGPU_OK;
}

}  // namespace bk

// bkgpu_host.hpp — C++ host side above the C ABI (include/bkgpu.h): the operator interface of the
// reference, mirrored so that a BaikalDB maintainer (or a test) drives the GPU path exactly the way
// Region::select drives any ExecNode (src/store/region.cpp:3069-3216):
//
//      ExecNode::create_tree -> root->open(&state) -> while (!eos) root->get_next(&state, &batch, &eos) -> root->close(&state)
//
// Mirrors (names, argument meaning, error convention):
//   ExecNode::init/open/get_next/close, add_child/replace_child     include/exec/exec_node.h:79-153
//   RuntimeState (error_code/error_msg, is_cancelled, counters)      include/runtime/runtime_state.h:312-324
//   pb::Plan / pb::PlanNode / pb::Expr / pb::ExprNode (pre-order)    proto/plan.proto:495-511, proto/expr.proto:67-84
//   MockScanNode feeding synthetic rows into a tree                  test/test_window.cpp:117-125,257-262
// Batches are COLUMN batches (what Chunk / RowBatch::transfer_rowbatch_to_arrow produce in the vectorized engine,
// include/runtime/row_batch.h:182-201), not MemRows.  Header-only, C++17, links against libbkgpu.so.
#pragma once
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <utility>
#include <vector>
#include "../include/bkgpu.h"

namespace bkgpu {

// ---------------------------------------------------------------- plan description (pb::Plan mirror)
struct Expr {
    int node_type = 0, col_type = 0;
    std::vector<Expr> children;
    int tuple_id = 0, slot_id = 0;
    int64_t int_val = 0; double double_val = 0; bool bool_val = false;
    int fn_op = 0; std::string name; std::vector<int> arg_types; int return_type = 0;
    int final_slot_id = 0, intermediate_slot_id = 0;

    static Expr slot_ref(int tuple, int slot, int type) { Expr e; e.node_type = BK_SLOT_REF; e.col_type = type; e.tuple_id = tuple; e.slot_id = slot; return e; }
    static Expr int_literal(int64_t v) { Expr e; e.node_type = BK_INT_LITERAL; e.col_type = BK_INT64; e.int_val = v; return e; }
    static Expr double_literal(double v) { Expr e; e.node_type = BK_DOUBLE_LITERAL; e.col_type = BK_DOUBLE; e.double_val = v; return e; }
    static Expr null_literal() { Expr e; e.node_type = BK_NULL_LITERAL; e.col_type = BK_NULL_TYPE; return e; }
    // STRING_LITERAL (taken where it folds into a date/time image) and the typed date/time literals, whose int_val is the image (literal.h:95-114)
    static Expr string_literal(std::string s) { Expr e; e.node_type = BK_STRING_LITERAL; e.col_type = BK_STRING; e.name = std::move(s); return e; }
    static Expr datetime_literal(int node_type, int col_type, int64_t image) { Expr e; e.node_type = node_type; e.col_type = col_type; e.int_val = image; return e; }
    static Expr fn(int fn_op, const char* name, std::vector<Expr> args) { Expr e; e.node_type = BK_FUNCTION_CALL; e.fn_op = fn_op; e.name = name; e.children = std::move(args); return e; }
    static Expr predicate(int node_type, int fn_op, const char* name, std::vector<Expr> args) {
        Expr e; e.node_type = node_type; e.col_type = BK_BOOL; e.fn_op = fn_op; e.name = name; e.children = std::move(args); return e;
    }
    // AGG_EXPR: name in {count_star,count,sum,avg,min,max}; intermediate != final only for AVG (expr.proto:59-60)
    static Expr agg(const char* name, int agg_tuple, int final_slot, int inter_slot, std::vector<Expr> args) {
        Expr e; e.node_type = BK_AGG_EXPR; e.name = name; e.tuple_id = agg_tuple; e.final_slot_id = final_slot; e.intermediate_slot_id = inter_slot;
        e.children = std::move(args); return e;
    }
    int count() const { int n = 1; for (auto& c : children) n += c.count(); return n; }
};

struct PlanNode {
    int node_type = 0;
    int64_t limit = -1;
    std::vector<PlanNode> children;
    int tuple_id = 0; int64_t table_id = 0;              // SCAN / SORT
    std::vector<Expr> conjuncts;                         // FILTER / JOIN / APPLY conditions
    int agg_tuple_id = -1; std::vector<Expr> group_exprs, agg_fn_calls;
    std::vector<Expr> order_exprs; std::vector<bool> is_asc, is_null_first;
    int join_type = BK_INNER_JOIN; int64_t offset = 0;
    bool max_one_row = false, is_select_field = false; int compare_type = BK_CMP_NULL;   // APPLY (its conditions in conjuncts)
    int count() const { int n = 1; for (auto& c : children) n += c.count(); return n; }
};

struct TupleDescriptor { int tuple_id; std::vector<std::pair<int, int>> slots; /* (slot_id, pb::PrimitiveType) */ };

class PlanWriter {   // the word stream of include/bkgpu_plan.h
public:
    std::vector<uint8_t> bytes;
    void w(int32_t v) { put(&v, 4); }
    void w64(int64_t v) { put(&v, 8); }
    void f64(double v) { put(&v, 8); }
    void str(const std::string& s) { w((int32_t)s.size()); put(s.data(), s.size()); static const char z[4] = {0, 0, 0, 0}; put(z, (4 - s.size() % 4) % 4); }
    void expr(const Expr& e) { w(e.count()); enode(e); }
    void node(const PlanNode& n) {
        w(n.node_type); w((int32_t)n.children.size()); w64(n.limit);
        switch (n.node_type) {
            case BK_SCAN_NODE: w(n.tuple_id); w64(n.table_id); break;
            case BK_WHERE_FILTER_NODE: case BK_TABLE_FILTER_NODE: case BK_HAVING_FILTER_NODE:
                w((int32_t)n.conjuncts.size()); for (auto& e : n.conjuncts) expr(e); break;
            case BK_AGG_NODE: case BK_MERGE_AGG_NODE:
                w(n.agg_tuple_id); w((int32_t)n.group_exprs.size()); for (auto& e : n.group_exprs) expr(e);
                w((int32_t)n.agg_fn_calls.size()); for (auto& e : n.agg_fn_calls) expr(e); break;
            case BK_SORT_NODE:
                w(n.tuple_id); w((int32_t)n.order_exprs.size());
                for (size_t i = 0; i < n.order_exprs.size(); i++) { expr(n.order_exprs[i]); w(n.is_asc[i] ? 1 : 0); w(n.is_null_first[i] ? 1 : 0); }
                break;
            case BK_JOIN_NODE: w(n.join_type); w((int32_t)n.conjuncts.size()); for (auto& e : n.conjuncts) expr(e); break;
            case BK_APPLY_NODE:
                w(n.join_type); w((int32_t)n.conjuncts.size()); for (auto& e : n.conjuncts) expr(e);
                w(n.max_one_row ? 1 : 0); w(n.compare_type); w(n.is_select_field ? 1 : 0); break;
            case BK_LIMIT_NODE: w64(n.offset); break;
            default: break;   // PACKET / SELECT_MANAGER: no payload
        }
        for (auto& c : n.children) node(c);
    }
private:
    void put(const void* p, size_t n) { const uint8_t* b = (const uint8_t*)p; bytes.insert(bytes.end(), b, b + n); }
    void enode(const Expr& e) {
        w(e.node_type); w(e.col_type); w((int32_t)e.children.size());
        switch (e.node_type) {
            case BK_SLOT_REF: w(e.tuple_id); w(e.slot_id); break;
            case BK_NULL_LITERAL: break;
            case BK_BOOL_LITERAL: w(e.bool_val ? 1 : 0); break;
            case BK_INT_LITERAL: w64(e.int_val); break;
            case BK_DOUBLE_LITERAL: f64(e.double_val); break;
            case BK_STRING_LITERAL: str(e.name); break;
            case BK_DATETIME_LITERAL: case BK_TIMESTAMP_LITERAL: case BK_DATE_LITERAL: case BK_TIME_LITERAL: w64(e.int_val); break;
            case BK_AGG_EXPR: str(e.name); w(e.tuple_id); w(e.final_slot_id); w(e.intermediate_slot_id); break;
            default: w(e.fn_op); str(e.name); w((int32_t)e.arg_types.size()); for (int a : e.arg_types) w(a); w(e.return_type); break;
        }
        for (auto& c : e.children) enode(c);
    }
};

struct Plan {
    std::vector<TupleDescriptor> tuples;   // sorted by tuple_id
    PlanNode root;
    std::vector<uint8_t> serialize() const {
        PlanWriter out;
        out.w((int32_t)BKGPU_PLAN_MAGIC); out.w(BKGPU_PLAN_VERSION); out.w((int32_t)tuples.size()); out.w(root.count());
        for (auto& t : tuples) { out.w(t.tuple_id); out.w((int32_t)t.slots.size()); for (auto& s : t.slots) { out.w(s.first); out.w(s.second); } }
        out.node(root);
        return out.bytes;
    }
};

// ---------------------------------------------------------------- batches and state
struct Column {
    int tuple_id = 0, slot_id = 0, prim_type = 0, elem_size = 0;
    std::vector<uint8_t> values;
    std::vector<uint8_t> validity;   // Arrow LSB bitmap; empty = no NULLs
    int64_t length = 0;
    template <class T> static Column from(int tuple, int slot, int prim, const std::vector<T>& v) {
        Column c; c.tuple_id = tuple; c.slot_id = slot; c.prim_type = prim; c.elem_size = (int)sizeof(T); c.length = (int64_t)v.size();
        c.values.resize(v.size() * sizeof(T)); if (!v.empty()) memcpy(c.values.data(), v.data(), c.values.size()); return c;
    }
    template <class T> T at(int64_t i) const { T v; memcpy(&v, values.data() + (size_t)i * sizeof(T), sizeof(T)); return v; }
    bool is_null(int64_t i) const { return !validity.empty() && !((validity[(size_t)i >> 3] >> (i & 7)) & 1); }
};

struct RowBatch {   // include/runtime/row_batch.h: here a batch of columns
    std::vector<Column> columns;
    int64_t size() const { return columns.empty() ? 0 : columns[0].length; }
    void clear() { columns.clear(); }
};

struct RuntimeState {
    int device = 0;
    void* nccl_comm = nullptr;
    int64_t row_batch_capacity = 1 << 20;
    int error_code = 0; std::string error_msg;
    int64_t num_scan_rows = 0, num_filter_rows = 0;
    bool cancelled = false;
    void cancel() { cancelled = true; }
    bool is_cancelled() const { return cancelled; }
};

// ---------------------------------------------------------------- rows <-> columns (f1: the MemRow / RowBatch bridge)
// What `MemRow::get_value(tuple, slot)` hands an operator: a typed value or NULL (include/mem_row/mem_row.h:28-215,
// ExprValue in include/common/expr_value.h).  64-bit payload in the slot's value class; an HLL sketch (BK_HLL: hll_add_agg's RAW sketch
// of 16400 bytes) is held as bytes, the way ExprValue holds it in str_val.
struct Value {
    bool is_null = true;
    union { int64_t i64; uint64_t u64; double f64; };
    std::string bytes;   // BK_HLL only
    Value() : i64(0) {}
    static Value of_int(int64_t v) { Value x; x.is_null = false; x.i64 = v; return x; }
    static Value of_uint(uint64_t v) { Value x; x.is_null = false; x.u64 = v; return x; }
    static Value of_double(double v) { Value x; x.is_null = false; x.f64 = v; return x; }
    static Value of_bytes(std::string v) { Value x; x.is_null = false; x.bytes = std::move(v); return x; }
};
using MemRowValues = std::vector<Value>;   // one Value per slot of the chunk's schema, in schema order

// Chunk: row -> column builder with the reference's type map (src/runtime/chunk.cpp:33-92: INT8/16/32,TIME -> int32;
// INT64 -> int64; UINT8/16/32,TIMESTAMP,DATE -> uint32; UINT64,DATETIME -> uint64; FLOAT -> f32; DOUBLE -> f64; BOOL -> u8)
class Chunk {
public:
    struct Slot { int tuple_id, slot_id, prim_type; };
    explicit Chunk(std::vector<Slot> schema) : _schema(std::move(schema)) { reset(); }
    static int storage_bytes(int prim) {
        switch (prim) {
            case BK_BOOL: return 1;
            case BK_INT8: case BK_INT16: case BK_INT32: case BK_TIME: case BK_UINT8: case BK_UINT16: case BK_UINT32: case BK_TIMESTAMP: case BK_DATE: case BK_FLOAT: return 4;
            case BK_INT64: case BK_UINT64: case BK_DATETIME: case BK_DOUBLE: return 8;
            case BK_HLL: return 16400;   // a RAW sketch (bkgpu.h)
            default: return -1;
        }
    }
    int add_row(const MemRowValues& row) {   // Chunk::add_row / decode_row (chunk.cpp:335-384)
        if (row.size() != _schema.size()) return -1;
        for (size_t c = 0; c < _schema.size(); c++)   // (a sketch of another length would shift every later row)
            if (_schema[c].prim_type == BK_HLL && !row[c].is_null && row[c].bytes.size() != (size_t)_batch.columns[c].elem_size) return -1;
        for (size_t c = 0; c < _schema.size(); c++) {
            Column& col = _batch.columns[c];
            const Value& v = row[c];
            const int eb = col.elem_size;
            const size_t off = col.values.size();
            col.values.resize(off + (size_t)eb, 0);
            if (v.is_null) {
                if (col.validity.empty()) col.validity.assign((size_t)(_rows + 8) / 8, 0xFF);
                if (col.validity.size() * 8 <= (size_t)_rows) col.validity.resize((size_t)_rows / 8 + 1, 0xFF);
                col.validity[(size_t)_rows >> 3] &= (uint8_t)~(1u << (_rows & 7));
            } else {
                if (!col.validity.empty() && col.validity.size() * 8 <= (size_t)_rows) col.validity.resize((size_t)_rows / 8 + 1, 0xFF);
                uint8_t* dst = col.values.data() + off;
                switch (_schema[c].prim_type) {
                    case BK_FLOAT: { float f = (float)v.f64; memcpy(dst, &f, 4); } break;
                    case BK_DOUBLE: memcpy(dst, &v.f64, 8); break;
                    case BK_BOOL: dst[0] = v.i64 ? 1 : 0; break;
                    case BK_HLL: memcpy(dst, v.bytes.data(), (size_t)eb); break;
                    default: memcpy(dst, &v.i64, (size_t)eb); break;   // little-endian narrowing of the integer payload
                }
            }
            col.length = _rows + 1;
        }
        _rows++;
        return 0;
    }
    int64_t size() const { return _rows; }
    RowBatch finish() {   // Chunk::finish_and_make_record_batch
        for (auto& c : _batch.columns) if (!c.validity.empty()) c.validity.resize((size_t)(_rows + 7) / 8 + 1, 0xFF);
        RowBatch out = std::move(_batch); reset(); return out;
    }
    // column batch -> rows (what a parent row-engine operator pulls out of a GPU subtree)
    static std::vector<MemRowValues> to_rows(const RowBatch& b) {
        std::vector<MemRowValues> rows((size_t)b.size(), MemRowValues(b.columns.size()));
        for (size_t c = 0; c < b.columns.size(); c++) {
            const Column& col = b.columns[c];
            for (int64_t r = 0; r < col.length; r++) {
                if (col.is_null(r)) continue;
                Value& v = rows[(size_t)r][c]; v.is_null = false;
                const uint8_t* src = col.values.data() + (size_t)r * (size_t)col.elem_size;
                switch (col.prim_type) {
                    case BK_FLOAT: { float f; memcpy(&f, src, 4); v.f64 = f; } break;
                    case BK_DOUBLE: memcpy(&v.f64, src, 8); break;
                    case BK_BOOL: v.i64 = src[0]; break;
                    case BK_INT8: case BK_INT16: case BK_INT32: case BK_TIME: { int32_t x; memcpy(&x, src, 4); v.i64 = x; } break;
                    case BK_UINT8: case BK_UINT16: case BK_UINT32: case BK_TIMESTAMP: case BK_DATE: { uint32_t x; memcpy(&x, src, 4); v.u64 = x; } break;
                    case BK_STRING: memcpy(&v.f64, src, 8); break;   // AVG intermediate: the sum half (count: src + 8)
                    case BK_HLL: v.bytes.assign((const char*)src, (size_t)col.elem_size); break;
                    default: memcpy(&v.i64, src, 8); break;
                }
            }
        }
        return rows;
    }
private:
    void reset() {
        _rows = 0; _batch.columns.clear();
        for (auto& s : _schema) { Column c; c.tuple_id = s.tuple_id; c.slot_id = s.slot_id; c.prim_type = s.prim_type; c.elem_size = storage_bytes(s.prim_type); _batch.columns.push_back(std::move(c)); }
    }
    std::vector<Slot> _schema; RowBatch _batch; int64_t _rows = 0;
};

// ---------------------------------------------------------------- operators
class ExecNode {
public:
    virtual ~ExecNode() = default;
    virtual int init(const Plan&) { return 0; }
    virtual int open(RuntimeState* state) { for (auto& c : _children) { int rc = c->open(state); if (rc < 0) return rc; } return 0; }
    virtual int get_next(RuntimeState* state, RowBatch* batch, bool* eos) = 0;
    virtual void close(RuntimeState* state) { for (auto& c : _children) c->close(state); }
    void add_child(std::unique_ptr<ExecNode> c) { _children.push_back(std::move(c)); }
    void replace_child(size_t i, std::unique_ptr<ExecNode> c) { _children[i] = std::move(c); }   // ExecNode::replace_child
protected:
    std::vector<std::unique_ptr<ExecNode>> _children;
};

// leaf: a scan that hands out prepared column batches (the MockScanNode of test/test_window.cpp:117-125)
class ColumnScanNode : public ExecNode {
public:
    explicit ColumnScanNode(std::vector<RowBatch> batches) : _batches(std::move(batches)) {}
    int get_next(RuntimeState*, RowBatch* batch, bool* eos) override {
        batch->clear();
        if (_pos < _batches.size()) *batch = std::move(_batches[_pos++]);
        *eos = _pos >= _batches.size();
        return 0;
    }
private:
    std::vector<RowBatch> _batches; size_t _pos = 0;
};

// leaf of a ROW engine below a GPU subtree: rows arrive one by one (RocksdbScanNode::get_next fills a RowBatch of <= 1024
// MemRows, include/runtime/row_batch.h:24-231); the Chunk turns every `capacity` of them into one column batch
class RowScanNode : public ExecNode {
public:
    RowScanNode(std::vector<Chunk::Slot> schema, std::vector<MemRowValues> rows, int64_t capacity = 1024)
        : _chunk(std::move(schema)), _rows(std::move(rows)), _capacity(capacity) {}
    int get_next(RuntimeState*, RowBatch* batch, bool* eos) override {
        batch->clear();
        while (_pos < _rows.size() && _chunk.size() < _capacity) if (_chunk.add_row(_rows[_pos++]) < 0) return -1;
        if (_chunk.size() > 0) *batch = _chunk.finish();
        *eos = _pos >= _rows.size();
        return 0;
    }
private:
    Chunk _chunk; std::vector<MemRowValues> _rows; size_t _pos = 0; int64_t _capacity;
};

// why this mirror cannot run a serialized plan ("" = it can): its Column holds fixed-width values, so a plan that returns rb_build_agg's
// variable-length BITMAP column is refused when the node is initialised (the C API and the Python binding return it)
inline std::string host_refusal(const std::vector<uint8_t>& plan) {
    std::string text(1 << 16, '\0');
    if (bkgpu_plan_explain(plan.data(), plan.size(), &text[0], text.size()) < 0) return "";   // (bkgpu_init reports a plan that does not lower)
    if (text.find("rb_build_agg: rb=") == std::string::npos) return "";
    return "rb_build_agg returns a BITMAP column, which the C++ host mirror does not carry: run the plan through the C API or the Python binding";
}

// the fused AGG -> [FILTER] -> SCAN / SORT / AGG -> JOIN / FILTER subtree on the GPU
class GpuExecNode : public ExecNode {
public:
    ~GpuExecNode() override { if (_h) bkgpu_close(_h); }
    int init(const Plan& plan) override { return init_serialized(plan.serialize()); }
    int init_serialized(std::vector<uint8_t> plan) {   // BKGPU_EUNSUPPORTED for a plan this mirror cannot carry; open() reports why
        _plan = std::move(plan);
        _refusal = host_refusal(_plan);
        return _refusal.empty() ? 0 : BKGPU_EUNSUPPORTED;
    }
    int open(RuntimeState* state) override {
        if (!_refusal.empty()) { state->error_code = BKGPU_EUNSUPPORTED; state->error_msg = _refusal; return -1; }
        int rc = bkgpu_init(&_h, _plan.data(), _plan.size(), state->device, state->nccl_comm);
        if (rc != 0) return fail(state, rc, nullptr);
        if ((rc = bkgpu_set_option(_h, "batch_capacity", state->row_batch_capacity)) != 0 || (rc = bkgpu_open(_h)) != 0) return fail(state, rc, _h);
        for (auto& child : _children) {   // children in driver-table-first order (the join's outer child is child 0)
            if (child->open(state) < 0) return -1;
            bool eos = false;
            while (!eos) {                 // the child-pull loop of AggNode::open (agg_node.cpp:447-485)
                if (state->is_cancelled()) { bkgpu_cancel(_h); return 0; }
                RowBatch b;
                if (child->get_next(state, &b, &eos) < 0) return -1;
                if (b.columns.empty()) continue;
                std::vector<bkgpu_column> cols(b.columns.size());
                for (size_t i = 0; i < cols.size(); i++) {
                    const Column& c = b.columns[i];
                    cols[i] = bkgpu_column{c.tuple_id, c.slot_id, c.prim_type, c.elem_size, c.values.data(), c.validity.empty() ? nullptr : c.validity.data(), c.length};
                }
                if ((rc = bkgpu_push(_h, cols.data(), (int)cols.size(), b.size(), 0)) != 0) return fail(state, rc, _h);
            }
        }
        if ((rc = bkgpu_finish(_h)) != 0) return fail(state, rc, _h);
        bkgpu_stats st; bkgpu_get_stats(_h, &st);
        state->num_scan_rows += st.rows_scanned; state->num_filter_rows += st.rows_filtered;   // region.cpp:3140-3143
        return 0;
    }
    int get_next(RuntimeState* state, RowBatch* batch, bool* eos) override {
        batch->clear();
        if (state->is_cancelled()) { *eos = true; return 0; }
        bkgpu_column cols[64]; int ncols = 64; int64_t nrows = 0; int e = 0;
        int rc = bkgpu_get_next(_h, cols, &ncols, &nrows, &e);
        if (rc != 0) return fail(state, rc, _h);
        for (int i = 0; i < ncols; i++) {
            Column c; c.tuple_id = cols[i].tuple_id; c.slot_id = cols[i].slot_id; c.prim_type = cols[i].prim_type; c.elem_size = cols[i].elem_size; c.length = nrows;
            c.values.assign((const uint8_t*)cols[i].values, (const uint8_t*)cols[i].values + (size_t)nrows * (size_t)cols[i].elem_size);
            if (cols[i].validity) c.validity.assign(cols[i].validity, cols[i].validity + (nrows + 7) / 8);
            batch->columns.push_back(std::move(c));
        }
        *eos = e != 0;
        return 0;
    }
    void close(RuntimeState* state) override { if (_h) { bkgpu_close(_h); _h = nullptr; } ExecNode::close(state); }
private:
    int fail(RuntimeState* state, int rc, bkgpu_plan* h) { state->error_code = rc; state->error_msg = bkgpu_last_error(h); return -1; }   // negative return + message
    std::vector<uint8_t> _plan;
    std::string _refusal;
    bkgpu_plan* _h = nullptr;
};

}  // namespace bkgpu

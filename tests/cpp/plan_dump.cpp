// Host-side dump of a plan's complete lowering: compile_plan over a plan descriptor, then every field of Compiled, its post and jfast
// fragments included.  The explain text prints the main program alone; this prints every program handed to the device.
//   g++ -std=c++17 -I csrc -I include -I /usr/local/cuda/include tests/cpp/plan_dump.cpp csrc/plan.cpp csrc/literal.cpp
//   plan_dump PLAN_FILE...
// Prints, per file, "== PLAN_FILE", rc, err and (rc == 0) the dump.
#include <inttypes.h>
#include <stdarg.h>
#include <stdio.h>
#include <string>
#include <vector>
#include "plan.h"
using namespace bk;

static void line(const std::string& ind, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
static void line(const std::string& ind, const char* fmt, ...) {
    fputs(ind.c_str(), stdout);
    va_list ap; va_start(ap, fmt); vprintf(fmt, ap); va_end(ap);
    fputc('\n', stdout);
}

template <class T> static std::string list(const std::vector<T>& v) {
    std::string s = "[";
    for (size_t i = 0; i < v.size(); i++) s += (i ? "," : "") + std::to_string((long long)v[i]);
    return s + "]";
}
template <class T> static std::string bytes(const T* v, int n) {   // a fixed-size array without its trailing zeros
    while (n > 0 && !v[n - 1]) n--;
    std::string s = "[";
    for (int i = 0; i < n; i++) s += (i ? "," : "") + std::to_string((int)v[i]);
    return s + "]";
}

// instructions, the constants up to the highest one an instruction uses (or the last one set), the NULL mask
template <class T> static bool zero(const T& v) {
    const unsigned char* b = (const unsigned char*)&v;
    for (size_t i = 0; i < sizeof v; i++) if (b[i]) return false;
    return true;
}

static void dump_program(const std::string& ind, const char* name, const Program& p) {
    if (zero(p)) { line(ind, "%s: zero", name); return; }
    line(ind, "%s: n_instr=%d n_out=%d cnull=0x%" PRIx64, name, p.n_instr, p.n_out, p.cnull);
    int n_const = 0;
    std::string code;
    for (int i = 0; i < p.n_instr && i < MAX_INSTR; i++) {
        const Instr& in = p.code[i];
        char buf[32];
        snprintf(buf, sizeof buf, "%s%d:%d,%d,%d", i ? " " : "", in.op, in.a, in.b, in.c);
        code += buf;
        int hi = -1;
        if (in.op == OP_CONST || in.op == OP_IN_SET) hi = in.a;
        if (in.op == OP_IN) hi = in.a + in.b - 1;
        if (in.op == OP_MATH && in.a == MF_ROUND) hi = in.b;
        if (hi + 1 > n_const) n_const = hi + 1;
    }
    for (int i = 0; i < MAX_CONST; i++) if ((p.cbits[i] || ((p.cnull >> i) & 1)) && i + 1 > n_const) n_const = i + 1;
    line(ind, "  code: %s", code.c_str());
    std::string k;
    for (int i = 0; i < n_const; i++) { char buf[24]; snprintf(buf, sizeof buf, "%s%" PRIx64, i ? " " : "", p.cbits[i]); k += buf; }
    line(ind, "  const: %s", k.c_str());
}

static void dump_agg_plan(const std::string& ind, const AggPlan& a) {
    if (zero(a)) { line(ind, "ap: zero"); return; }
    line(ind, "ap: n_keyw=%d n_group=%d n_agg=%d n_lanes=%d pred_out=%d", a.n_keyw, a.n_group, a.n_agg, a.n_lanes, a.pred_out);
    line(ind, "  lane_op=%s", bytes(a.lane_op, MAX_LANES).c_str());
    line(ind, "  key_out=%s key_word=%s key_shift=%s key_bits=%s", bytes(a.key_out, MAX_GROUP).c_str(), bytes(a.key_word, MAX_GROUP).c_str(),
         bytes(a.key_shift, MAX_GROUP).c_str(), bytes(a.key_bits, MAX_GROUP).c_str());
    line(ind, "  key_null_word=%s key_null_shift=%s key_prim=%s", bytes(a.key_null_word, MAX_GROUP).c_str(), bytes(a.key_null_shift, MAX_GROUP).c_str(),
         bytes(a.key_prim, MAX_GROUP).c_str());
    for (int k = 0; k < MAX_AGG; k++) {
        const AggSpec& s = a.agg[k];
        if (k >= a.n_agg && zero(s)) continue;
        line(ind, "  agg[%d] kind=%d vclass=%d acc_lane=%d cnt_lane=%d arg_out=%d nullable=%d out_prim=%d arg_vclass=%d cnt_owner=%d acc_owner=%d hidden=%d", k, s.kind,
             s.vclass, s.acc_lane, s.cnt_lane, s.arg_out, s.nullable, s.out_prim, s.arg_vclass, s.cnt_owner, s.acc_owner, s.hidden);
    }
}

static void dump_direct(const std::string& ind, const DirectPlan& d) {
    if (zero(d)) { line(ind, "direct: zero"); return; }
    line(ind, "direct: n_terms=%d n_keys=%d n_vals=%d key_col=%s val_col=%s agg_val=%s", d.n_terms, d.n_keys, d.n_vals, bytes(d.key_col, 2).c_str(),
         bytes(d.val_col, 8).c_str(), bytes(d.agg_val, MAX_AGG).c_str());
    for (int t = 0; t < 4; t++)
        if (t < d.n_terms || !zero(d.term[t])) line(ind, "  term[%d] col=%d cmp=%d vclass=%d cbits=%" PRIx64, t, d.term[t].col, d.term[t].cmp, d.term[t].vclass, d.term[t].cbits);
}

static uint64_t fnv1a(const std::vector<uint64_t>& v) {
    uint64_t h = 1469598103934665603ull;
    for (uint64_t w : v) for (int b = 0; b < 8; b++) { h ^= (w >> (8 * b)) & 0xFF; h *= 1099511628211ull; }
    return h;
}

static bool same_tuples(const std::vector<HTuple>& a, const std::vector<HTuple>& b) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); i++) if (a[i].tuple_id != b[i].tuple_id || a[i].slots != b[i].slots) return false;
    return true;
}

static const Compiled* g_root;

static void dump(const Compiled& c, const std::string& ind, const InSets* root_sets, bool root) {
    line(ind, "kind=%d scan_tuple=%d build_tuple=%d", c.kind, c.scan_tuple, c.build_tuple);
    if (!root && same_tuples(c.tuples, g_root->tuples)) line(ind, "tuples: the plan's");
    else for (auto& t : c.tuples) {
        std::string s;
        for (auto& sl : t.slots) s += " " + std::to_string(sl.first) + ":" + std::to_string(sl.second);
        line(ind, "tuple %d:%s", t.tuple_id, s.c_str());
    }
    for (size_t i = 0; i < c.cols.size(); i++)
        line(ind, "col[%zu] %d_%d prim=%d side=%d", i, c.cols[i].tuple_id, c.cols[i].slot_id, c.cols[i].prim, i < c.col_side.size() ? c.col_side[i] : -99);
    if (c.col_side.size() != c.cols.size()) line(ind, "col_side size %zu != cols size %zu", c.col_side.size(), c.cols.size());
    for (size_t i = 0; i < c.out_cols.size(); i++)
        line(ind, "out_col[%zu] %d_%d prim=%d kind=%d", i, c.out_cols[i].tuple_id, c.out_cols[i].slot_id, c.out_cols[i].prim, c.out_cols[i].kind);
    for (auto& k : c.sort_keys) line(ind, "sort_key out_reg=%d prim=%d asc=%d null_first=%d", k.out_reg, k.prim, (int)k.asc, (int)k.null_first);
    line(ind, "limit=%" PRId64 " offset=%" PRId64 " agg_limit=%" PRId64, c.limit, c.offset, c.agg_limit);
    line(ind, "is_merge=%d emit_default=%d has_direct=%d direct_cols=%s", (int)c.is_merge, (int)c.emit_default, (int)c.has_direct, list(c.direct_cols).c_str());
    std::vector<int> can_null(c.arg_can_null.begin(), c.arg_can_null.end());
    line(ind, "arg_cols_mask=%s arg_can_null=%s", list(c.arg_cols_mask).c_str(), list(can_null).c_str());
    line(ind, "join: type=%d key_prim=%d build_key_col=%d probe_key_col=%d n_build_filter=%d n_probe_filter=%d", c.join_type, c.join_key_prim, c.build_key_col,
         c.probe_key_col, c.n_build_filter, c.n_probe_filter);
    dump_program(ind, "prog", c.prog);
    dump_agg_plan(ind, c.ap);
    dump_direct(ind, c.direct);
    dump_program(ind, "build_filter", c.build_filter);
    dump_program(ind, "probe_filter", c.probe_filter);
    for (size_t k = 0; k < c.dims.size(); k++) {
        const StarDim& d = c.dims[k];
        line(ind, "dim[%zu] tuple=%d key_col=%d fk_col=%d cast_prim=%d n_filter=%d", k, d.tuple_id, d.key_col, d.fk_col, d.cast_prim, d.n_filter);
        dump_program(ind + "  ", "filter", d.filter);
    }
    for (size_t k = 0; k < c.win.size(); k++) {
        const WinStage& w = c.win[k];
        line(ind, "win[%zu] new_sort=%d n_part=%d has_frame=%d frame_type=%d start=%d,%d,%" PRId64 " end=%d,%d,%" PRId64 " expr_prim=%s", k, (int)w.new_sort, w.n_part,
             (int)w.has_frame, w.frame_type, w.start.type, (int)w.start.unbounded, w.start.num, w.end.type, (int)w.end.unbounded, w.end.num, list(w.expr_prim).c_str());
        for (auto& sk : w.sort_keys) line(ind, "  sort_key out_reg=%d prim=%d asc=%d null_first=%d", sk.out_reg, sk.prim, (int)sk.asc, (int)sk.null_first);
        for (auto& f : w.fns)
            line(ind, "  fn kind=%d %d_%d out_prim=%d arg=%d def=%d arg_prim=%d n=%" PRId64 " method=%d", f.kind, f.tuple_id, f.slot_id, f.out_prim, f.arg, f.def,
                 f.arg_prim, f.n, f.method);
        for (size_t i = 0; i < w.exprs.size(); i++) dump_program(ind + "  ", ("expr[" + std::to_string(i) + "]").c_str(), w.exprs[i]);
    }
    if (!c.in_sets) line(ind, "in_sets: none");
    else if (!root && c.in_sets.get() == root_sets) line(ind, "in_sets: the plan's");
    else {
        line(ind, "in_sets: %s", root ? "plan" : "own");
        for (size_t i = 0; i < c.in_sets->sets.size(); i++) {
            const InSet& s = c.in_sets->sets[i];
            line(ind, "  set[%zu] vclass=%d has_null=%d n_distinct=%u words=%zu hash=%016" PRIx64, i, s.vclass, (int)s.has_null, s.n_distinct, s.image.size(), fnv1a(s.image));
        }
        std::vector<int> idx;
        for (auto& x : c.in_sets->of_expr) idx.push_back(x.second);
        line(ind, "  of_expr=%s", list(idx).c_str());
    }
    line(ind, "jfast_of_main=%s", list(c.jfast_of_main).c_str());
    if (c.jfast) { line(ind, "jfast:"); dump(*c.jfast, ind + "    ", root_sets, false); }
    if (c.post) { line(ind, "post:"); dump(*c.post, ind + "    ", root_sets, false); }
    if (!c.explain.empty()) {
        line(ind, "explain:");
        fputs(c.explain.c_str(), stdout);
    }
}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: %s PLAN_FILE...\n", argv[0]); return 2; }
    for (int a = 1; a < argc; a++) {
        std::vector<uint8_t> desc;
        FILE* fp = fopen(argv[a], "rb");
        if (!fp) { perror(argv[a]); return 2; }
        for (int ch; (ch = fgetc(fp)) != EOF;) desc.push_back((uint8_t)ch);
        fclose(fp);
        Compiled c{};
        std::string err;
        const int rc = compile_plan(desc.data(), desc.size(), c, err);
        printf("== %s\nrc=%d\nerr=%s\n", argv[a], rc, err.c_str());
        g_root = &c;
        if (rc == 0) dump(c, "", c.in_sets.get(), true);
    }
    return 0;
}

// Host-side check of the aggregate kernel choice (csrc/agg_select.cpp): compiles a plan descriptor, builds one batch of device
// columns with fake pointers (the choice reads a pointer only for its alignment), runs select_agg_launch and prints what it chose.
//   g++ -std=c++17 -I csrc -I include -I /usr/local/cuda/include tests/cpp/agg_select_check.cpp csrc/agg_select.cpp csrc/plan.cpp csrc/literal.cpp
//   agg_select_check PLAN_FILE [name=value ...]
// Batch: valid=COLS (columns with a validity bitmap), offset=COL:BYTES (values that many bytes past a 4 KB boundary), vec_ok=0|1,
// nrows=N, known_groups=G, fused=1 (the fused FK -> PK probe: the join's fast-path plan, a mode-1 JoinProbe).  COLS are plan columns
// named tuple_slot, comma-separated.  Every other name is an AggEnv field.  Prints one name=value per line.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "agg_select.h"
#include "bkgpu.h"
using namespace bk;

static const char* const kKernels[] = {"INTERP", "SCALAR_DIRECT", "COUNT_WHERE_TMA", "GROUP_DIRECT", "LEAN", "LEAN_NULLS", "LEAN_MM",
                                       "LEAN_FX", "LEAN_JOIN", "LEAN_FX_JOIN"};

static int col_index(const Compiled& c, const std::string& name) {
    for (size_t i = 0; i < c.cols.size(); i++)
        if (std::to_string(c.cols[i].tuple_id) + "_" + std::to_string(c.cols[i].slot_id) == name) return (int)i;
    fprintf(stderr, "no plan column %s\n", name.c_str());
    exit(2);
}

static std::vector<std::string> split(const std::string& s, char sep) {
    std::vector<std::string> out;
    size_t a = 0;
    for (size_t b; (b = s.find(sep, a)) != std::string::npos; a = b + 1) out.push_back(s.substr(a, b - a));
    out.push_back(s.substr(a));
    return out;
}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: %s PLAN_FILE [name=value ...]\n", argv[0]); return 2; }
    std::vector<uint8_t> desc;
    {
        FILE* fp = fopen(argv[1], "rb");
        if (!fp) { perror(argv[1]); return 2; }
        for (int ch; (ch = fgetc(fp)) != EOF;) desc.push_back((uint8_t)ch);
        fclose(fp);
    }
    Compiled c;
    std::string err;
    if (compile_plan(desc.data(), desc.size(), c, err) != 0) { fprintf(stderr, "compile_plan: %s\n", err.c_str()); return 2; }

    // the plan object's defaults
    AggEnv env;
    env.scalar_tma = 1; env.lean_fx = BK_LEAN_FX_DEFAULT; env.smem_cap_log2 = -1;
    env.has_post = c.post != nullptr;
    int64_t nrows = 1 << 20;
    bool vec_ok = true, fused = false;
    std::vector<DevCol> cols(c.cols.size());
    for (size_t i = 0; i < cols.size(); i++) {
        cols[i].values = (const void*)(uintptr_t)((i + 1) << 20);
        cols[i].validity = nullptr;
        cols[i].stype = prim_storage(c.cols[i].prim);
        cols[i].prim = c.cols[i].prim;
    }
    struct { const char* name; int* field; } ints[] = {
        {"force_generic", &env.force_generic}, {"no_lean", &env.no_lean}, {"no_lean_nulls", &env.no_lean_nulls}, {"no_lean_mm", &env.no_lean_mm},
        {"lean_fx", &env.lean_fx}, {"fx_off", &env.fx_off}, {"scalar_tma", &env.scalar_tma}, {"smem_cap_log2", &env.smem_cap_log2}};
    for (int k = 2; k < argc; k++) {
        const std::string arg = argv[k];
        const size_t eq = arg.find('=');
        if (eq == std::string::npos) { fprintf(stderr, "bad argument %s\n", argv[k]); return 2; }
        const std::string name = arg.substr(0, eq), val = arg.substr(eq + 1);
        const long long v = atoll(val.c_str());
        bool known = true;
        if (name == "valid") { for (auto& s : split(val, ',')) cols[(size_t)col_index(c, s)].validity = (const uint8_t*)(uintptr_t)(0x40000000u + (col_index(c, s) << 20)); }
        else if (name == "offset") { auto f = split(val, ':'); DevCol& d = cols[(size_t)col_index(c, f.at(0))]; d.values = (const uint8_t*)d.values + atoi(f.at(1).c_str()); }
        else if (name == "vec_ok") vec_ok = v != 0;
        else if (name == "nrows") nrows = v;
        else if (name == "known_groups") env.known_groups = (uint32_t)v;
        else if (name == "fused") fused = v != 0;
        else if (name == "tail_launch") env.tail_launch = v != 0;
        else if (name == "multi_rank") env.multi_rank = v != 0;
        else {
            known = false;
            for (auto& f : ints) if (name == f.name) { *f.field = (int)v; known = true; }
        }
        if (!known) { fprintf(stderr, "unknown argument %s\n", argv[k]); return 2; }
    }

    // the fused probe runs the join's fast-path plan over the probe row: its key column is the probe-side foreign key (join.cu)
    const Compiled* plan = &c;
    JoinProbe jp{};
    if (fused) {
        if (!c.jfast || !c.jfast->has_direct) { fprintf(stderr, "the plan has no fused probe\n"); return 2; }
        const Compiled& f = *c.jfast;
        std::vector<DevCol> fc(f.cols.size());
        const int key_fcol = f.direct_cols[(size_t)f.direct.n_terms];
        for (size_t i = 0; i < f.cols.size(); i++) fc[i] = (int)i == key_fcol ? cols[(size_t)c.probe_key_col] : cols[(size_t)c.jfast_of_main[i]];
        cols = fc;
        plan = &f;
        jp.mode = 1; jp.key_signed = 1; jp.dense_size = 1000;
    }

    AggArgs a;
    AggSelection sel;
    const int rc = select_agg_launch(*plan, cols.data(), nrows, vec_ok, fused ? &jp : nullptr, env, a, sel);
    printf("rc=%d\n", rc);
    if (rc) return 0;
    printf("kernel=%s\nname=%s\nsmem=%zu\nfused_ok=%d\n", kKernels[sel.kernel], agg_kernel_name(sel.kernel), sel.smem, sel.fused_ok ? 1 : 0);
    printf("smem_cap_log2=%d\nn_smem_lanes=%d\nsmem_lane=", a.smem_cap_log2, a.n_smem_lanes);
    for (int l = 0; l < a.plan.n_lanes; l++) printf(l ? ",%d" : "%d", a.smem_lane[l] == 0xFF ? -1 : (int)a.smem_lane[l]);
    printf("\nlean=%d\nlean_fx=%d\nfx_ext_off=%u\n", a.lean, a.lean_fx, a.fx_ext_off);
    return 0;
}

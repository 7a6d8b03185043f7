// agg_select.cpp — the choice of the aggregate kernel for one batch (see agg_select.h).  Pure host code: the launchers in agg.cu,
// scalar_tma.cu and agg_direct.cuh dispatch on its AggKernel and decide nothing themselves.
#include "agg_select.h"
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include "../include/bkgpu.h"
#include "../include/bkgpu_plan.h"

namespace bk {

const char* agg_kernel_name(AggKernel k) {
    switch (k) {
        case INTERP: return "k_agg_interp";
        case SCALAR_DIRECT: return "k_agg_scalar_direct";
        case COUNT_WHERE_TMA: return "k_count_where_tma";
        case GROUP_DIRECT: return "k_agg_group_direct";
        case LEAN_FX: case LEAN_FX_JOIN: return "k_agg_group_lean_fx";
        default: return "k_agg_group_lean";
    }
}

size_t agg_smem_bytes(int smem_keyw, int n_smem_lanes, int cap_log2) {
    if (cap_log2 <= 0 || smem_keyw == 0) return 0;
    return ((size_t)(smem_keyw + n_smem_lanes) * 8 + 4) << cap_log2;
}

// shared memory of the direct GROUP BY kernel: the table plus one compaction queue per warp
size_t direct_smem_bytes(int smem_keyw, int n_smem_lanes, int cap_log2, int na) {
    const size_t table = (agg_smem_bytes(smem_keyw, n_smem_lanes, cap_log2) + 127) & ~(size_t)127;
    const size_t q_direct = ((size_t)(2 + na) * 128 + 16) * 8;  // QCAP = 128 entries per warp, up to 2 key words
    const size_t q_lean = ((((size_t)(1 + na) * 160 + 20) + 15) & ~(size_t)15) * 8 + 8;   // LEAN_QCAP = 160-entry ring, one key word, 128-byte aligned (+ slack for the base)
    const size_t queue = q_direct > q_lean ? q_direct : q_lean;
    const int warps = (DIRECT_THREADS > LEAN_THREADS ? DIRECT_THREADS : LEAN_THREADS) / 32;   // sized for the larger of the two CTA shapes
    return table + queue * warps;
}

// FX (agg_direct.cuh): one low-extension limb (4 bytes) per value column and slot, behind the queues
size_t fx_ext_bytes(int na, int cap_log2) { return ((size_t)4 * (size_t)na) << cap_log2; }

// the shape of k_count_where_tma: COUNT(*) only, WHERE one NULL-free, 16-byte aligned int32 column <cmp> an int32 constant
static bool count_where_tma_shape(const AggArgs& a) {
    if (a.plan.n_keyw != 0 || a.direct.n_terms != 1 || a.direct.n_vals != 0 || a.plan.n_agg < 1) return false;
    for (int k = 0; k < a.plan.n_agg; k++) if (a.plan.agg[k].kind != AG_COUNT_STAR) return false;
    const DevCol& c = a.cols[0];
    const DirectTerm& tm = a.direct.term[0];
    const int64_t cv = (int64_t)tm.cbits;
    return c.stype == ST_I32 && c.prim == BK_INT32 && !c.validity && tm.vclass == VC_I64 && cv >= INT32_MIN && cv <= INT32_MAX && ((uintptr_t)c.values & 15) == 0;
}

// the shared-table capacity for this batch: >= 2x the groups seen so far, 2048 slots when nothing is known yet, 0 (straight to the global
// table) when the groups cannot fit one CTA's 227 KB
static int pick_smem_log2(const AggEnv& env, int n_keyw, int n_smem_lanes, bool direct, int na) {
    if (n_keyw == 0) return 0;
    const size_t budget = 220 * 1024;
    auto bytes = [&](int log2) { return direct ? direct_smem_bytes(n_keyw, n_smem_lanes, log2, na) : agg_smem_bytes(n_keyw, n_smem_lanes, log2); };
    if (env.smem_cap_log2 >= 0) { int l = env.smem_cap_log2; while (l > 0 && bytes(l) > budget) l--; return l; }
    const uint32_t g = env.known_groups;
    int log2 = 11;
    while (((uint32_t)1 << log2) < 2 * g && log2 < 14) log2++;
    while (log2 > 0 && bytes(log2) > budget) log2--;
    if (((uint32_t)1 << log2) < g) return 0;  // would mostly miss: skip the shared table
    return log2;
}

// does a direct batch fit the lean kernel?  `mm`: some column feeds MIN / MAX or several lanes (the MM instantiation)
static bool lean_fits(const Compiled& c, const AggArgs& a, bool nulls_ok, bool mm_ok, bool& mm) {
    const int np = c.direct.n_terms, na = c.direct.n_vals;
    bool any_valid = false;
    for (int i = 0; i < a.n_cols; i++) if (a.cols[i].validity) any_valid = true;
    bool ok = !a.cols[np].validity && (!any_valid || nulls_ok);   // NULL keys (and NULLs under the fused probe) take the general kernel
    for (int t = 0; t < np && ok; t++) {
        const DirectTerm& tm = c.direct.term[t];
        const int64_t cv = (int64_t)tm.cbits;
        ok = a.cols[t].stype == ST_I32 && a.cols[t].prim == BK_INT32 && tm.vclass == VC_I64 && cv >= INT32_MIN && cv <= INT32_MAX;
    }
    const DevCol& kc = a.cols[np];
    ok = ok && ((kc.stype == ST_I32 && kc.prim == BK_INT32) || (kc.stype == ST_U32 && kc.prim == BK_UINT32) || kc.stype == ST_I64 || kc.stype == ST_U64);
    mm = false;
    for (int v = 0; v < na && ok; v++) {
        const DevCol& vc = a.cols[np + 1 + v];
        const ValOps& vo = a.vops[v];
        ok = (vc.stype == ST_F64 || vc.stype == ST_I64 || vc.stype == ST_U64) && vo.n_ops <= 3 && (vo.cnt_smem == 0xFF || vo.cnt_glob != 0);
        const int col_class = vc.stype == ST_F64 ? VC_F64 : (vc.stype == ST_U64 ? VC_U64 : VC_I64);
        for (int k = 0; k < vo.n_ops && ok; k++) {
            const int op = vo.op[k];
            if (op == LN_ADD_F64) ok = vc.stype == ST_F64 && vo.lane_class[k] == VC_F64;
            else if (op == LN_ADD_I64) ok = vc.stype != ST_F64;
            else { ok = vo.lane_class[k] == col_class && vo.arg_class == col_class; mm = true; }   // MIN / MAX in the column's own class
        }
        if (vo.n_ops != 1) mm = true;
    }
    return ok && (!mm || mm_ok);
}

int select_agg_launch(const Compiled& c, const DevCol* cols, int64_t nrows, bool vec_ok, const JoinProbe* jp, const AggEnv& env, AggArgs& a,
                      AggSelection& out) {
    out = AggSelection{};
    memset(&a, 0, sizeof a);
    a.plan = c.ap; a.prog = c.prog; a.direct = c.direct;
    const bool direct = c.has_direct && vec_ok && !env.force_generic && c.kind == PK_AGG && !c.ap.n_hll && !c.n_rb;   // (the join's fast-path plan is lowered as PK_AGG)
    const int ncols = (int)c.cols.size();
    if (direct) { for (size_t i = 0; i < c.direct_cols.size(); i++) a.cols[i] = cols[c.direct_cols[i]]; a.n_cols = (int)c.direct_cols.size(); }
    else { for (int i = 0; i < ncols; i++) a.cols[i] = cols[i]; a.n_cols = ncols; }
    // per-batch nullability -> which lanes need per-row work in the shared table
    memset(a.smem_lane, 0xFF, sizeof a.smem_lane);
    a.smem_lane[0] = 0; a.n_smem_lanes = 1; a.alias_mask = 0;
    for (int k = 0; k < a.plan.n_agg; k++) {
        AggSpec& s = a.plan.agg[k];
        if (s.kind == AG_COUNT_STAR || s.kind == AG_RB) continue;   // (AG_RB: no lane; its keys go to the pair buffer)
        bool nullable = c.arg_can_null[(size_t)k] || env.tail_launch;   // (the tail's probe-side columns are NULL on every row)
        for (int i = 0; i < ncols; i++) if ((c.arg_cols_mask[(size_t)k] >> i) & 1) nullable = nullable || cols[i].validity != nullptr;
        s.nullable = nullable ? 1 : 0;
        if (s.cnt_lane && s.cnt_owner) {
            if (nullable) { if (a.smem_lane[s.cnt_lane] == 0xFF) a.smem_lane[s.cnt_lane] = (uint8_t)a.n_smem_lanes++; }
            else a.alias_mask |= 1u << s.cnt_lane;
        }
        if (s.kind != AG_COUNT && a.smem_lane[s.acc_lane] == 0xFF) a.smem_lane[s.acc_lane] = (uint8_t)a.n_smem_lanes++;
    }
    for (int l = 1; l < a.plan.n_lanes; l++) if (a.smem_lane[l] != 0xFF) a.alias_mask &= ~(1u << l);
    a.smem_cap_log2 = c.ap.n_hll || c.n_rb ? 0 : pick_smem_log2(env, a.plan.n_keyw, a.n_smem_lanes, direct, c.direct.n_vals);   // (a sketch lives in the global table's arena, a pair in its buffer: both need the global slot)
    a.smem_sentinel = direct && a.plan.n_keyw == 1 ? 1 : 0;
    a.smem_keyw = a.plan.n_keyw;

    if (direct) {  // per value column: the lane operations it feeds
        memset(a.vops, 0, sizeof a.vops);
        for (int v = 0; v < c.direct.n_vals; v++) { a.vops[v].cnt_smem = 0xFF; }
        for (int k = 0; k < a.plan.n_agg; k++) {
            const AggSpec& s = a.plan.agg[k];
            if (s.kind == AG_COUNT_STAR) continue;
            ValOps& vo = a.vops[c.direct.agg_val[k]];
            vo.arg_class = s.arg_vclass;
            if (s.cnt_lane && s.cnt_owner) { vo.cnt_glob = s.cnt_lane; vo.cnt_smem = s.nullable ? a.smem_lane[s.cnt_lane] : 0xFF; }
            if (s.kind != AG_COUNT && s.acc_owner) {
                const int n = vo.n_ops++;
                vo.op[n] = a.plan.lane_op[s.acc_lane]; vo.lane_class[n] = s.vclass; vo.glob_lane[n] = s.acc_lane; vo.smem_lane[n] = a.smem_lane[s.acc_lane];
            }
        }
    }
    a.lean = 0;
    // lean shape: one key word, or a 64-bit key whose second word only carries the (here unused) NULL flag
    const bool lean_keyw = a.plan.n_keyw == 1 || (a.plan.n_keyw == 2 && a.plan.n_group == 1 && a.plan.key_bits[0] == 64 && a.plan.key_null_word[0] == 1);
    bool mm = false;
    if (direct && lean_keyw && a.smem_cap_log2 > 0 && !env.no_lean && lean_fits(c, a, !jp && !env.no_lean_nulls, !jp && !env.no_lean_mm, mm)) {
        const int na = c.direct.n_vals;
        bool any_valid = false;
        for (int i = 0; i < a.n_cols; i++) if (a.cols[i].validity) any_valid = true;
        a.lean = 1;
        a.smem_sentinel = 1; a.smem_keyw = 1; a.smem_paired = 1;
        // lane placement for 128-bit shared CAS: ONE double sum shares a 16-byte word with the row count
        // ({rows, sum}: a single atomic per row); otherwise double sums sit in pairs {sumA, sumB}
        memset(a.smem_lane, 0xFF, sizeof a.smem_lane);
        a.smem_lane[0] = 0;
        int nf64 = 0;   // columns that feed exactly one double sum (they sit in {sumA, sumB} pairs)
        for (int v = 0; v < na; v++) if (a.vops[v].n_ops == 1 && a.vops[v].op[0] == LN_ADD_F64) nf64++;
        int next_f = nf64 == 1 ? 1 : 2, next_i = nf64 == 1 ? 2 : 2 + ((nf64 + 1) & ~1);
        for (int v = 0; v < na; v++) {
            ValOps& vo = a.vops[v];
            for (int k = 0; k < vo.n_ops; k++) {
                const int sl = (vo.n_ops == 1 && vo.op[0] == LN_ADD_F64) ? next_f++ : next_i++;
                vo.smem_lane[k] = (uint8_t)sl; a.smem_lane[vo.glob_lane[k]] = (uint8_t)sl;
            }
        }
        a.lean_mm = mm ? 1 : 0;
        int next = std::max(next_f, next_i);
        for (int v = 0; v < na; v++) {   // non-NULL counters of the value columns that carry NULLs in this batch
            ValOps& vo = a.vops[v];
            if (vo.cnt_smem == 0xFF) continue;
            vo.cnt_smem = (uint8_t)next; a.smem_lane[vo.cnt_glob] = (uint8_t)next; next++;
        }
        a.lean_nulls = any_valid ? 1 : 0;
        a.n_smem_lanes = (next + 1) & ~1;
        if (a.n_smem_lanes < 2) a.n_smem_lanes = 2;
        a.smem_cap_log2 = pick_smem_log2(env, a.plan.n_keyw, a.n_smem_lanes, true, na);
        if (a.smem_cap_log2 <= 0) { a.lean = 0; a.smem_paired = 0; return BKGPU_ENOMEM; }
        // FX: plain batches (no NULLs, no MIN / MAX) with at least one double sum, when the extension limbs fit beside table and queues
        if (env.lean_fx && !env.fx_off && !mm && !any_valid && nf64 >= 1 && nrows < ((int64_t)1 << 31)) {
            const size_t base = direct_smem_bytes(a.smem_keyw, a.n_smem_lanes, a.smem_cap_log2, na);
            if (base + fx_ext_bytes(na, a.smem_cap_log2) <= (size_t)224 * 1024) { a.lean_fx = 1; a.fx_ext_off = (uint32_t)base; }   // (227 KB per CTA less the kernel's 1 KB of static shared memory)
        }
    }
    if (jp) { if (!a.lean) return 1; a.jp = *jp; }
    a.scalar_tma = env.scalar_tma;

    const bool grouped = a.plan.n_keyw > 0;
    const int na = c.direct.n_vals;
    if (!direct) out.kernel = INTERP;
    else if (!grouped) out.kernel = env.scalar_tma && count_where_tma_shape(a) ? COUNT_WHERE_TMA : SCALAR_DIRECT;
    else if (!a.lean) out.kernel = GROUP_DIRECT;
    else if (a.lean_mm) out.kernel = LEAN_MM;   // (one MM / NULLS instantiation serves batches with and without NULLs)
    else if (a.lean_nulls) out.kernel = LEAN_NULLS;
    else if (a.lean_fx) out.kernel = a.jp.mode ? LEAN_FX_JOIN : LEAN_FX;
    else if (a.jp.mode) out.kernel = LEAN_JOIN;
    else out.kernel = LEAN;
    if (!grouped || out.kernel == COUNT_WHERE_TMA) out.smem = 0;
    else if (!direct) out.smem = agg_smem_bytes(a.smem_keyw, a.n_smem_lanes, a.smem_cap_log2);
    else out.smem = direct_smem_bytes(a.smem_keyw, a.n_smem_lanes, a.smem_cap_log2, na) + (a.lean_fx ? fx_ext_bytes(na, a.smem_cap_log2) : 0);
    // a lean launch on one rank whose rows go straight to the host extracts its own result: any of them may be the request's last
    out.fused_ok = direct && a.lean && grouped && !env.multi_rank && !env.has_post;
    return BKGPU_OK;
}

}  // namespace bk

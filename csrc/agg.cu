// agg.cu — K1+K2: fused scan -> filter -> (GROUP BY) aggregate kernels for sm_90a.
//
// Replaces, for one column batch, the reference's hot loop
//     AggNode::open:  do { child->get_next(batch); process_row_batch(batch); } while (!eos)
//         /root/reference/src/exec/agg_node.cpp:447-485,507-545
// with its per-row FilterNode::need_copy (src/exec/filter_node.cpp:726-734), ExecNode::encode_exprs_key
// (src/exec/exec_node.cpp:555-571) and AggFnCall::update (src/expr/agg_fn_call.cpp:496-555).
//
// Data flow: every referenced column is read exactly once with 256-bit non-allocating loads
// (8 rows per thread and load); the predicate is evaluated in registers; passing rows update a
// per-CTA open-addressed hash table in shared memory (native 32-bit ATOMS for counts, CAS loop for
// double sums); each CTA merges its table once into the global group table (RED.ADD.F64 / RED.ADD.64).
// Rows whose group does not fit the shared table go straight to the global table, so any
// cardinality is handled; the global table is also the per-GPU partial state that NCCL ships.
//
// This file holds the generic (interpreted) kernel, the join probe loops that run the interpreter, the group table's maintenance,
// exchange and extraction kernels, and the aggregate's host path: the group table's allocation, the launch of each batch, the
// exchange between ranks and the result (agg_open / agg_push / agg_finish / agg_reset / agg_partial_*, declared in api_state.h).
// The lean and direct kernels are agg_direct.cuh's.
#include <string.h>
#include <algorithm>
#include <vector>
#include "agg_kernels.cuh"
#include "interp.cuh"
#include "agg_select.h"
#include "api_state.h"
#include "nccl_dl.h"
#include "prims.cuh"

namespace bk {

// ------------------------------------------------------------------------------------------
// generic path: the lowered expression program (interp.cuh) is interpreted per row (any predicate,
// computed keys and arguments, multi-column keys).
// ------------------------------------------------------------------------------------------
// the AG_HLL aggregates of one row that reached group `slot` (out of line: the other plans' interpreter keeps its registers)
static __device__ __noinline__ void hll_row(const AggArgs& a, const uint64_t* out, uint32_t out_null, int slot) {
    const AggPlan& ap = a.plan;
    for (int i = 0; i < ap.n_agg; i++) {
        const AggSpec s = ap.agg[i];
        if (s.kind != AG_HLL || ((out_null >> s.arg_out) & 1u)) continue;
        if (s.arg_prim == BK_HLL) hll_merge_value(a.gt, s, a.cols[s.hll_col], (int64_t)out[s.arg_out], a.gt.lanes, a.gt.cap_mask + 1, slot);
        else hll_add_value(a.gt, s, a.gt.lanes, a.gt.cap_mask + 1, slot, out[s.arg_out]);
    }
}
// the AG_RB aggregates of one row that reached group `slot`: each non-NULL argument appends its pair key (AggArgs::rb_keys) with one
// atomic per warp.  rb_build_agg adds get_numberic<uint32_t>(value): the low 32 bits of the integer image (agg_fn_call.cpp:642-651)
static __device__ __noinline__ void rb_row(const AggArgs& a, const uint64_t* out, uint32_t out_null, int slot) {
    const AggPlan& ap = a.plan;
    const int lane = threadIdx.x & 31;
    for (int i = 0; i < ap.n_agg; i++) {
        const AggSpec s = ap.agg[i];
        if (s.kind != AG_RB) continue;
        const bool has = !((out_null >> s.arg_out) & 1u);
        const unsigned m = __ballot_sync(__activemask(), has);
        if (!has) continue;
        const int leader = __ffs(m) - 1;
        unsigned long long base = 0;
        if (lane == leader) base = atomicAdd(a.rb_ctr, (unsigned long long)__popc(m));
        base = __shfl_sync(m, base, leader);
        const unsigned long long pos = base + (unsigned long long)__popc(m & ((1u << lane) - 1u));
        if (pos < a.rb_cap) a.rb_keys[pos] = ((uint64_t)slot << 34) | ((uint64_t)s.rb_idx << 32) | (uint32_t)out[s.arg_out];
    }
}
// one (possibly joined) row through the program into the tables
struct InterpCtx { SmemTable st; bool grouped, use_smem; uint32_t gcap; };
// how: 0 = filter, then aggregate the row; 1 = filter only (SEMI / ANTI probe: does the joined row satisfy the conditions?);
//      2 = aggregate without the filter (the NULL-extended / preserved rows of the join's tail)
// MODE: IM_HLL = the plan has AG_HLL aggregates, IM_RB = AG_RB aggregates (IM_PLAIN keeps the interpreter's registers as they were)
enum InterpMode { IM_PLAIN = 0, IM_HLL = 1, IM_RB = 2 };
template <int MODE = IM_PLAIN>
__device__ __forceinline__ uint32_t interp_row(const AggArgs& a, const InterpCtx& cx, int64_t row, int64_t brow, int how = 0) {
    const AggPlan& ap = a.plan;
    const GroupTable& gt = a.gt;
    uint64_t out[MAX_GROUP + MAX_AGG + 1];
    uint32_t out_null;
    run_program(a.prog, a.cols, row, out, out_null, brow);
    if (how != 2 && ap.pred_out >= 0 && (((out_null >> ap.pred_out) & 1u) || out[ap.pred_out] == 0)) return 0;
    if (how == 1) return 1;
    auto arg = [&](int i, uint64_t& v, bool& isnull) {
        const int r = ap.agg[i].arg_out;
        if (r == 0xFF) { v = 0; isnull = true; return; }
        v = out[r]; isnull = (out_null >> r) & 1u;
    };
    // hll_add_agg / rb_build_agg (such a plan never uses the shared table: a sketch lives in the global table's arena, a pair in its buffer)
    auto sketch = [&](int slot) { if (MODE == IM_HLL) hll_row(a, out, out_null, slot); else if (MODE == IM_RB) rb_row(a, out, out_null, slot); };
    if (!cx.grouped) {  // single group: slot 0 of the global table
        accumulate_row<false>(a, gt.lanes, cx.gcap, 0, arg);
        sketch(0);
        return 1;
    }
    uint64_t key[MAX_KEYW];
    for (int w = 0; w < ap.n_keyw; w++) key[w] = 0;
    for (int g = 0; g < ap.n_group; g++) {
        const int r = ap.key_out[g];
        if ((out_null >> r) & 1u) key[ap.key_null_word[g]] |= 1ull << ap.key_null_shift[g];
        else {
            const uint64_t m = ap.key_bits[g] >= 64 ? ~0ull : ((1ull << ap.key_bits[g]) - 1ull);
            key[ap.key_word[g]] |= (out[r] & m) << ap.key_shift[g];
        }
    }
    const uint32_t h = ap.n_keyw == 1 ? hash_key1(key[0]) : hash_key(key, ap.n_keyw);
    int slot = -1;
    if (cx.use_smem) slot = table_upsert<true, 0>(cx.st.state, cx.st.keys, cx.st.cap_mask, key, ap.n_keyw, h >> 7, 16, nullptr);
    if (slot >= 0) accumulate_row<true>(a, cx.st.lanes, cx.st.cap_mask + 1, slot, arg);
    else {
        slot = table_upsert<false, 0>(gt.state, gt.keys, gt.cap_mask, key, ap.n_keyw, h, (int)cx.gcap, gt.n_groups);
        if (slot < 0) atomicExch(gt.overflow, 1u);
        else { accumulate_row<false>(a, gt.lanes, cx.gcap, slot, arg); sketch(slot); }
    }
    return 1;
}

template <int MODE>
__global__ void __launch_bounds__(256) k_agg_interp(const __grid_constant__ AggArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const AggPlan& ap = a.plan;
    InterpCtx cx;
    cx.grouped = ap.n_keyw > 0;
    cx.use_smem = cx.grouped && a.smem_cap_log2 > 0;
    cx.gcap = a.gt.cap_mask + 1;
    cx.st = SmemTable{};
    if (cx.use_smem) cx.st = smem_table_init(smem_raw, a);
    uint32_t passed = 0;
    if (a.join.enabled && a.join.tail) {   // after the last probe batch: the preserved (build) side's rows the join type asks for
        const int jt = a.join.join_type;
        for (int64_t br = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; br < a.join.n_build; br += (int64_t)gridDim.x * blockDim.x) {
            const uint8_t m = a.join.matched[br];   // (2: removed by the build side's own filter, never emitted)
            if (jt == 4 /*SEMI*/ ? m == 1 : m == 0) passed += interp_row<MODE>(a, cx, -1, br, 2);
        }
    } else
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < a.nrows; row += (int64_t)gridDim.x * blockDim.x) {
        if (!a.join.enabled) { passed += interp_row<MODE>(a, cx, row, -1); continue; }
        // K4 probe: every build row whose cast key equals this row's (Joiner::encode_hash_key + FlatMap seek,
        // src/exec/joiner.cpp:608-622, join_node.cpp:1290-1292); a NULL key never matches (SQL / Acero hashjoin)
        const DevCol& pc = a.cols[a.join.probe_col];
        if (elem_is_null(pc, row)) continue;
        const uint64_t img = cast_prim(load_elem(pc, row), a.join.probe_prim, a.join.cast_prim);
        uint32_t slot = hash_key1(img) & a.join.cap_mask;
        for (;;) {
            const uint32_t br = a.join.rows[slot];
            if (br == 0xFFFFFFFFu) break;
            if (a.join.keys[slot] == img) {
                if (a.join.join_type == 3 /*INNER*/ || !a.join.matched) passed += interp_row<MODE>(a, cx, row, (int64_t)br);
                else if (a.join.join_type == 1 /*LEFT*/) { if (interp_row<MODE>(a, cx, row, (int64_t)br)) { passed++; a.join.matched[br] = 1; } }
                else if (interp_row(a, cx, row, (int64_t)br, 1)) a.join.matched[br] = 1;   // SEMI / ANTI_SEMI: only whether a partner exists
            }
            slot = (slot + 1) & a.join.cap_mask;
        }
    }
    if (cx.use_smem) smem_table_flush(cx.st, a);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) passed += __shfl_xor_sync(0xFFFFFFFFu, passed, d);
    if ((threadIdx.x & 31) == 0 && passed) atomicAdd((unsigned long long*)a.rows_passed, (unsigned long long)passed);
}

// ---- a JOIN that returns rows (JoinNode::get_next_for_hash_inner_join / _other_join, join_node.cpp:1200-1326): the probe emits (probe row,
// build row) pairs, a gather per output column follows.  LEFT: matched[] is set here, the tail emits (NONE, build row) for the rest.
__global__ void __launch_bounds__(256) k_join_pairs(const __grid_constant__ AggArgs a, uint32_t* pairs, uint32_t cap, uint32_t* cursor) {
    InterpCtx cx; cx.grouped = false; cx.use_smem = false; cx.gcap = 0; cx.st = SmemTable{};
    auto emit = [&](uint32_t prow, uint32_t brow) {
        const uint32_t pos = atomicAdd(cursor, 1u);
        if (pos < cap) { pairs[2 * (size_t)pos] = prow; pairs[2 * (size_t)pos + 1] = brow; }   // (past the capacity only the count matters: the host grows the buffer and reruns)
    };
    if (a.join.tail) {
        for (int64_t br = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; br < a.join.n_build; br += (int64_t)gridDim.x * blockDim.x)
            if (a.join.matched[br] == 0) emit(JOIN_NO_ROW, (uint32_t)br);
        return;
    }
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < a.nrows; row += (int64_t)gridDim.x * blockDim.x) {
        const DevCol& pc = a.cols[a.join.probe_col];
        if (elem_is_null(pc, row)) continue;
        const uint64_t img = cast_prim(load_elem(pc, row), a.join.probe_prim, a.join.cast_prim);
        uint32_t slot = hash_key1(img) & a.join.cap_mask;
        for (;;) {
            const uint32_t br = a.join.rows[slot];
            if (br == 0xFFFFFFFFu) break;
            if (a.join.keys[slot] == img && interp_row(a, cx, row, (int64_t)br, 1)) {
                if (a.join.matched) a.join.matched[br] = 1;
                emit((uint32_t)row, br);
            }
            slot = (slot + 1) & a.join.cap_mask;
        }
    }
}
// FULL (Acero's FULL_OUTER hashjoin with the residual conditions as its filter, join_node.cpp:857-875): a probe row leaves one pair per partner
// that satisfies the conditions (setting matched[]), or one (row, JOIN_NO_ROW) when none does — a NULL key included.  Every probe row emits,
// so output slots are reserved per warp and round (ballot + one cursor atomic) rather than per pair.  Same capacity contract as k_join_pairs;
// the tail (unmatched build rows) is k_join_pairs' tail branch.
__global__ void __launch_bounds__(256) k_join_pairs_full(const __grid_constant__ AggArgs a, uint32_t* pairs, uint32_t cap, uint32_t* cursor) {
    InterpCtx cx; cx.grouped = false; cx.use_smem = false; cx.gcap = 0; cx.st = SmemTable{};
    const int lane = threadIdx.x & 31;
    const uint32_t lt = (1u << lane) - 1u;
    const DevCol& pc = a.cols[a.join.probe_col];
    for (int64_t w0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); w0 < a.nrows; w0 += (int64_t)gridDim.x * blockDim.x) {   // (warp-uniform: the ballots)
        const int64_t row = w0 + lane;
        int state = 0;   // 0 = done, 1 = walking the multimap, 2 = no partner passed: the NULL-extended pair is due
        bool found = false;
        uint64_t img = 0; uint32_t slot = 0;
        if (row < a.nrows) {
            if (elem_is_null(pc, row)) state = 2;
            else { img = cast_prim(load_elem(pc, row), a.join.probe_prim, a.join.cast_prim); slot = hash_key1(img) & a.join.cap_mask; state = 1; }
        }
        for (;;) {   // one round: every lane emits at most one pair
            uint32_t br = JOIN_NO_ROW;
            bool emit = false;
            while (state == 1) {
                const uint32_t s = slot, r = a.join.rows[s];
                if (r == 0xFFFFFFFFu) { state = found ? 0 : 2; break; }
                slot = (slot + 1) & a.join.cap_mask;
                if (a.join.keys[s] == img && interp_row(a, cx, row, (int64_t)r, 1)) { a.join.matched[r] = 1; found = true; br = r; emit = true; break; }
            }
            if (state == 2) { emit = true; state = 0; }
            const uint32_t b = __ballot_sync(0xFFFFFFFFu, emit);
            if (!b) break;   // (a lane still walking always emits: no emitter means every lane is done)
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(cursor, (uint32_t)__popc(b));
            base = __shfl_sync(0xFFFFFFFFu, base, 0);
            const uint32_t pos = base + (uint32_t)__popc(b & lt);
            if (emit && pos < cap) { pairs[2 * (size_t)pos] = (uint32_t)row; pairs[2 * (size_t)pos + 1] = br; }
        }
    }
}

// ------------------------------------------------------------------------------------------
// table maintenance: init, partial export / import (K3), result extraction + finalize
// ------------------------------------------------------------------------------------------
__global__ void k_table_init(GroupTable gt, AggPlan ap, int keep_overflow) {
    const uint32_t cap = gt.cap_mask + 1;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += gridDim.x * blockDim.x) {
        gt.state[i] = ap.n_keyw == 0 ? 2u : 0u;
        for (int l = 0; l < ap.n_lanes; l++) gt.lanes[(size_t)l * cap + i] = lane_identity(ap.lane_op[l]);
    }
    // (re-initialisation between the export of a partial state and the merge keeps the overflow flag: a table that overflowed
    //  while rows were pushed, or an export that met more groups than the exchange format holds, must still fail the plan)
    if (blockIdx.x == 0 && threadIdx.x < GT_OCC_OFF && !keep_overflow) gt.n_groups[threadIdx.x] = 0;   // fresh request: every counter of the block
    if (blockIdx.x == 0 && threadIdx.x == 0 && keep_overflow) *gt.n_groups = 0;                          // mid-request re-initialisation (multi-GPU merge): the group count only
    if (blockIdx.x == 0 && threadIdx.x < 3 && gt.hll_ctr && !(threadIdx.x >= 1 && keep_overflow)) gt.hll_ctr[threadIdx.x] = 0;   // (the sketch lanes are 0 again)
}

// walk the groups a table holds: the occupied list of a GROUP BY table (slots in insertion order), slot 0 of a scalar aggregate
#define BK_FOR_EACH_GROUP(gt, ap, i)                                                                                   \
    const uint32_t bk_n_ = (ap).n_keyw == 0 ? 1u : *(gt).n_groups;                                                    \
    for (uint32_t bk_j_ = blockIdx.x * blockDim.x + threadIdx.x, i = 0; bk_j_ < bk_n_ && ((i = (ap).n_keyw == 0 ? 0u : (gt).n_groups[GT_OCC_OFF + bk_j_]), true); bk_j_ += gridDim.x * blockDim.x)

// re-initialisation of a table whose `n` occupied slots are known (bkgpu_reset after a finished run): touches n slots, not the capacity
__global__ void k_table_clear(GroupTable gt, AggPlan ap, uint32_t n) {
    const uint32_t cap = gt.cap_mask + 1;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t i = gt.n_groups[GT_OCC_OFF + j];
        gt.state[i] = 0u;
        for (int l = 0; l < ap.n_lanes; l++) gt.lanes[(size_t)l * cap + i] = lane_identity(ap.lane_op[l]);
    }
    // (the counters can go in the same launch: nobody here reads them — `n` came by value, the occupied list sits behind them)
    if (blockIdx.x == 0 && threadIdx.x < GT_OCC_OFF) gt.n_groups[threadIdx.x] = 0;
    if (blockIdx.x == 0 && threadIdx.x < 3 && gt.hll_ctr) gt.hll_ctr[threadIdx.x] = 0;
}

// Compact partial state for the all-gather (the default multi-GPU merge): dst[0] = the number of groups this rank holds (its low
// half doubles as the export cursor, so it may exceed `bound`), followed by min(groups, bound) rows of n_keyw + n_lanes words.
// Only `1 + bound * row words` cross NVLink; `bound` follows the group counts seen in earlier runs (agg_collective).
__global__ void k_partial_export_rows(GroupTable gt, AggPlan ap, uint64_t* dst, uint32_t bound) {
    const uint32_t cap = gt.cap_mask + 1;
    const int rw = ap.n_keyw + ap.n_lanes + ap.n_hll * HLL_ROW_WORDS;
    BK_FOR_EACH_GROUP(gt, ap, i) {
        if (ap.n_keyw == 0 && gt.lanes[i] == 0) continue;  // no row reached the single group
        const uint32_t pos = atomicAdd((uint32_t*)dst, 1u);
        if (pos >= bound) continue;                         // (the merge sees count > bound and asks for a second, larger exchange)
        uint64_t* row = dst + 1 + (size_t)pos * rw;
        for (int w = 0; w < ap.n_keyw; w++) row[w] = gt.keys[(size_t)w * cap + i];
        for (int l = 0; l < ap.n_lanes; l++) row[ap.n_keyw + l] = gt.lanes[(size_t)l * cap + i];
        // each sketch's registers after the lanes, in aggregate order (all zero for a group without a value); its lane keeps only
        // whether the group has a sketch: 0 none, 1 a sketch, 2 one this table lost to a full arena (the merger fails too).  A block
        // index means nothing to another table
        uint64_t* regs_out = row + ap.n_keyw + ap.n_lanes;
        for (int k = 0; k < ap.n_agg; k++) {
            if (ap.agg[k].kind != AG_HLL) continue;
            const uint64_t ref = gt.lanes[(size_t)ap.agg[k].acc_lane * cap + i];
            row[ap.n_keyw + ap.agg[k].acc_lane] = ref == 0 ? 0 : ref >= HLL_LANE_FULL ? 2 : 1;
            const uint64_t* src = ref == 0 || ref >= HLL_LANE_FULL ? nullptr : (const uint64_t*)(gt.hll_regs + (size_t)(ref - 1) * HLL_REGISTERS);
            for (int w = 0; w < HLL_ROW_WORDS; w++) regs_out[w] = src ? __ldcg((const unsigned long long*)src + w) : 0ull;
            regs_out += HLL_ROW_WORDS;
        }
    }
}
// the sketches of an imported group row (k_partial_export_rows' layout) folded into the group at `slot`: register-wise max
__device__ __forceinline__ void hll_merge_row(const AggPlan& ap, const GroupTable& gt, int slot, const uint64_t* row) {
    const uint32_t cap = gt.cap_mask + 1;
    const uint64_t* regs_in = row + ap.n_keyw + ap.n_lanes;
    for (int k = 0; k < ap.n_agg; k++) {
        if (ap.agg[k].kind != AG_HLL) continue;
        const uint64_t has = row[ap.n_keyw + ap.agg[k].acc_lane];
        if (has == 2) atomicExch(gt.hll_ctr + 1, 1u);   // (the exporting table's arena overflowed: this sketch would be truncated)
        else if (has) {
            uint8_t* regs = hll_sketch(gt, gt.lanes + (size_t)ap.agg[k].acc_lane * cap + slot);
            if (regs)
                for (int w = 0; w < 2 * HLL_ROW_WORDS; w++) {
                    const unsigned int x = ((const unsigned int*)regs_in)[w];
                    if (x) hll_max_word((unsigned int*)regs + w, x, __ldcg((const unsigned int*)regs + w));
                }
        }
        regs_in += HLL_ROW_WORDS;
    }
}
// K3 on the gathered rows: every rank folds the OTHER ranks' groups into its own table (its own groups are already there), so
// nothing is re-initialised.  When some rank held more groups than `bound` nothing is merged anywhere (every rank reads the same
// headers) and *max_count tells the host to repeat the exchange with a larger bound.  A merge of exported buffers (self < 0,
// bkgpu_partial_merge) has no second exchange: a segment that holds more groups than its rows carry came from an export that failed
// with ETOOBIG, and the merge fails with it (the overflow flag) instead of returning the other segments' groups alone.
__global__ void k_partial_merge_rows(GroupTable gt, AggPlan ap, const uint64_t* src, size_t words_per_rank, uint32_t bound, int nranks, int self, uint32_t* max_count) {
    uint32_t mx = 0;
    for (int r = 0; r < nranks; r++) { const uint32_t c = (uint32_t)src[(size_t)r * words_per_rank]; mx = c > mx ? c : mx; }
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
        *max_count = mx;
        if (mx > bound && self < 0) atomicExch(gt.overflow, 1u);
    }
    if (mx > bound) return;
    const int r = blockIdx.y;
    if (r == self) return;
    const uint64_t* base = src + (size_t)r * words_per_rank;
    const uint32_t n = (uint32_t)base[0];
    const int rw = ap.n_keyw + ap.n_lanes + ap.n_hll * HLL_ROW_WORDS;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint64_t* row = base + 1 + (size_t)i * rw;
        uint64_t key[MAX_KEYW];
        for (int w = 0; w < ap.n_keyw; w++) key[w] = row[w];
        merge_group(ap, gt, key, [&](int l, uint64_t& v) { v = row[ap.n_keyw + l]; return ap.lane_op[l] != LN_HLL; });
        if (ap.n_hll) {   // the group's slot, which merge_group has just found or inserted
            const int slot = ap.n_keyw == 0 ? 0 : table_upsert<false, 0>(gt.state, gt.keys, gt.cap_mask, key, ap.n_keyw,
                                                                       ap.n_keyw == 1 ? hash_key1(key[0]) : hash_key(key, ap.n_keyw),
                                                                       (int)(gt.cap_mask + 1), gt.n_groups);
            if (slot >= 0) hll_merge_row(ap, gt, slot, row);
        }
    }
}

// hash repartition (the reference's exchange between fragments, src/exec/exchange_sender_node.cpp:867-957): every group of this
// rank's table goes to the segment of the rank that OWNS its key.  Segment layout (fixed capacity `pcap` groups):
// [u64 n_groups][keys n_keyw x pcap][lanes n_lanes x pcap]
__device__ __forceinline__ uint32_t owner_of(const uint64_t* key, int kw, int nranks) {
    uint64_t h = 0xC2B2AE3D27D4EB4Full;
    for (int i = 0; i < kw; i++) { h ^= key[i]; h *= 0x9FB21C651E98DF25ull; h ^= h >> 29; }
    return (uint32_t)((h >> 17) % (uint64_t)nranks);
}
__global__ void k_partial_export_parts(GroupTable gt, AggPlan ap, uint64_t* dst, size_t words_per_seg, uint32_t pcap, uint32_t* cursors, int nranks) {
    const uint32_t cap = gt.cap_mask + 1;
    BK_FOR_EACH_GROUP(gt, ap, i) {
        uint64_t key[MAX_KEYW];
        for (int w = 0; w < ap.n_keyw; w++) key[w] = gt.keys[(size_t)w * cap + i];
        const uint32_t o = owner_of(key, ap.n_keyw, nranks);
        const uint32_t pos = atomicAdd(cursors + o, 1u);
        if (pos >= pcap) { atomicExch(gt.overflow, 1u); continue; }
        uint64_t* dkeys = dst + (size_t)o * words_per_seg + 1;
        uint64_t* dlanes = dkeys + (size_t)ap.n_keyw * pcap;
        for (int w = 0; w < ap.n_keyw; w++) dkeys[(size_t)w * pcap + pos] = key[w];
        for (int l = 0; l < ap.n_lanes; l++) dlanes[(size_t)l * pcap + pos] = gt.lanes[(size_t)l * cap + i];
    }
}
__global__ void k_partial_counts(uint64_t* dst, size_t words_per_seg, const uint32_t* cursors, uint32_t pcap, int nranks) {
    const int r = threadIdx.x;
    if (r < nranks) dst[(size_t)r * words_per_seg] = cursors[r] < pcap ? cursors[r] : pcap;
}

// K3: fold `nranks` exported partials into the (re-initialised) global table
__global__ void k_partial_merge(GroupTable gt, AggPlan ap, const uint64_t* src, size_t words_per_rank, uint32_t pcap, int nranks) {
    for (int r = 0; r < nranks; r++) {
        const uint64_t* base = src + (size_t)r * words_per_rank;
        const uint32_t n = (uint32_t)base[0] < pcap ? (uint32_t)base[0] : pcap;   // (a count beyond the segment's capacity never indexes past it)
        const uint64_t* skeys = base + 1;
        const uint64_t* slanes = skeys + (size_t)ap.n_keyw * pcap;
        for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
            uint64_t key[MAX_KEYW];
            for (int w = 0; w < ap.n_keyw; w++) key[w] = skeys[(size_t)w * pcap + i];
            merge_group(ap, gt, key, [&](int l, uint64_t& v) { v = slanes[(size_t)l * pcap + i]; return true; });
        }
    }
}

// Result extraction: one output row per occupied slot (extract_group, agg_kernels.cuh), rows of stride out_cap.
__global__ void k_extract(GroupTable gt, AggPlan ap, uint64_t* outv, uint8_t* outn, uint32_t out_cap, uint32_t* cursor, int emit_default) {
    BK_FOR_EACH_GROUP(gt, ap, i) {
        if (ap.n_keyw == 0 && gt.lanes[i] == 0 && !emit_default) continue;
        const uint32_t pos = atomicAdd(cursor, 1u);
        if (pos >= out_cap) continue;
        extract_group(gt, ap, i, pos, outv, outn, out_cap);
    }
}

// The aggregate's extracted rows (canonical 64-bit images + null bytes, column-major with stride out_cap) as typed Arrow-layout
// columns on the device: the input of the post fragment ([LIMIT ->] [SORT ->] [HAVING ->] above the aggregate).
struct PostCols { int32_t n; int32_t img[MAX_COLS]; int32_t stype[MAX_COLS]; uint8_t* values[MAX_COLS]; uint8_t* null_bytes[MAX_COLS]; };
__global__ void k_images_to_columns(const uint64_t* outv, const uint8_t* outn, uint32_t out_cap, uint32_t n, PostCols pc) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        for (int c = 0; c < pc.n; c++) {
            const int img = pc.img[c];
            const uint64_t v = outv[(size_t)img * out_cap + r];
            pc.null_bytes[c][r] = outn[(size_t)img * out_cap + r];
            switch (pc.stype[c]) {
                case ST_I32: ((int32_t*)pc.values[c])[r] = (int32_t)(int64_t)v; break;
                case ST_U32: ((uint32_t*)pc.values[c])[r] = (uint32_t)v; break;
                case ST_F32: ((float*)pc.values[c])[r] = (float)bits_f64(v); break;
                case ST_U8: ((uint8_t*)pc.values[c])[r] = v ? 1 : 0; break;
                case ST_BLOB16: ((uint64_t*)pc.values[c])[2 * (size_t)r] = v; ((uint64_t*)pc.values[c])[2 * (size_t)r + 1] = outv[(size_t)(img + 1) * out_cap + r]; break;
                default: ((uint64_t*)pc.values[c])[r] = v; break;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// host-side launchers
// ------------------------------------------------------------------------------------------
template <class K>
static int occupancy_grid(K kernel, size_t smem, int sm_count) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    return per_sm * sm_count;  // persistent grid: a whole number of CTAs per SM (132 SMs on H100 SXM)
}

// the aggregate kernel `k` over one batch; `smem`: its dynamic shared memory (AggSelection::smem).  `start` (optional) is recorded on `s`
// right before the kernel launch, after the launch setup
static cudaError_t launch_agg(const AggArgs& a, AggKernel k, size_t smem, int sm_count, cudaStream_t s, cudaEvent_t start) {
    if (a.nrows <= 0) return cudaSuccess;
    switch (k) {
        case INTERP: {
            auto kern = a.gt.hll_regs ? k_agg_interp<IM_HLL> : a.rb_keys ? k_agg_interp<IM_RB> : k_agg_interp<IM_PLAIN>;
            if (smem > 48 * 1024) {
                cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
                if (e != cudaSuccess) return e;
            }
            int grid = occupancy_grid(kern, smem, sm_count);
            int64_t want = (a.nrows + 255) / 256;
            if (want < grid) grid = (int)want;
            if (start) cudaEventRecord(start, s);
            kern<<<grid, 256, smem, s>>>(a);
            return cudaGetLastError();
        }
        case COUNT_WHERE_TMA: return launch_count_where_tma(a, sm_count, s, start);
        default:
            switch (a.direct.n_terms) {
                case 0: return launch_direct_np0(a, k, sm_count, smem, s, start);
                case 1: return launch_direct_np1(a, k, sm_count, smem, s, start);
                default: return launch_direct_np2(a, k, sm_count, smem, s, start);
            }
    }
}

cudaError_t launch_join_pairs(const AggArgs& a, uint32_t* pairs, uint32_t cap, uint32_t* cursor, int sm_count, cudaStream_t s) {
    const int64_t n = a.join.tail ? a.join.n_build : a.nrows;
    if (n == 0) return cudaSuccess;
    int64_t g64 = (n + 255) / 256; if (g64 > (int64_t)sm_count * 8) g64 = (int64_t)sm_count * 8;
    const int grid = g64 < 1 ? 1 : (int)g64;
    if (a.join.join_type == 6 /*FULL*/ && !a.join.tail) k_join_pairs_full<<<grid, 256, 0, s>>>(a, pairs, cap, cursor);
    else k_join_pairs<<<grid, 256, 0, s>>>(a, pairs, cap, cursor);
    return cudaGetLastError();
}

}  // namespace bk

// ------------------------------------------------------------------------------------------
// host path of the aggregate (PK_AGG, PK_JOIN_AGG, PK_STAR_AGG): the group table, its launches, the exchange between ranks and
// the result
// ------------------------------------------------------------------------------------------
// record = false: the caller records ep->a itself (right before its launch)
static EventPair* timer_begin(bkgpu_plan* p, std::vector<EventPair>& v, int64_t bytes, bool record = true) {
    EventPair ep{};
    for (cudaEvent_t* e : {&ep.a, &ep.b}) {   // events are recycled: a re-armed plan launches the same kernels again and again
        if (!p->event_pool.empty()) { *e = p->event_pool.back(); p->event_pool.pop_back(); }
        else if (cudaEventCreate(e) != cudaSuccess) return nullptr;
    }
    ep.bytes = bytes;
    if (record) cudaEventRecord(ep.a, p->stream);
    v.push_back(ep);
    return &v.back();
}
static void timer_end(bkgpu_plan* p, EventPair* ep) { if (ep) cudaEventRecord(ep->b, p->stream); }

int agg_open(bkgpu_plan* p, AggState& g, const Compiled& c) {
    const AggPlan& ap = c.ap;
    GroupTable& gt = g.gt;
    if (cudaHostAlloc((void**)&g.h_pinned, 64, cudaHostAllocDefault) == cudaSuccess) memset(g.h_pinned, 0, 64); else g.h_pinned = nullptr;
    g.blocking_wait = g.blocking_sync >= 0 ? g.blocking_sync != 0 : (p->nranks > 1 && cpu_budget() < 4 * p->nranks);   // (agg_wait)
    int log2 = ap.n_keyw == 0 ? 0 : g.group_cap_log2;
    size_t cap = (size_t)1 << log2;
    gt.cap_mask = (uint32_t)(cap - 1); gt.cap_log2 = (uint32_t)log2;
    int rc;
    if ((rc = dev_alloc(p, (void**)&gt.state, cap * 4))) return rc;
    if ((rc = dev_alloc(p, (void**)&gt.keys, cap * 8 * (size_t)std::max(ap.n_keyw, 1)))) return rc;
    if ((rc = dev_alloc(p, (void**)&gt.lanes, cap * 8 * (size_t)ap.n_lanes))) return rc;
    if ((rc = dev_alloc(p, (void**)&gt.n_groups, 4 * ((size_t)GT_OCC_OFF + cap)))) return rc;   // counter, overflow flag, occupied list
    gt.overflow = gt.n_groups + 1;
    if (ap.n_hll) {   // hll_add_agg: the register arena, one block per (group, sketch) that receives a value
        if ((rc = dev_alloc(p, (void**)&gt.hll_regs, (size_t)g.hll_cap * HLL_REGISTERS))) return rc;
        if ((rc = dev_alloc(p, (void**)&gt.hll_ctr, 16))) return rc;
        gt.hll_cap = (uint32_t)g.hll_cap;
        CK(p, cudaMemsetAsync(gt.hll_ctr, 0, 16, p->stream));
    }
    if (c.n_rb) {   // rb_build_agg: the pair buffer and the sort's second buffer (one word more each: the build's scan closes on it)
        if ((rc = dev_alloc(p, (void**)&g.rb.keys, ((size_t)g.rb_cap + 1) * 8))) return rc;
        if ((rc = dev_alloc(p, (void**)&g.rb.alt, ((size_t)g.rb_cap + 1) * 8))) return rc;
        if ((rc = dev_alloc(p, (void**)&g.rb.ctr, 8))) return rc;
        g.rb.cap = (uint64_t)g.rb_cap;
        CK(p, cudaMemsetAsync(g.rb.ctr, 0, 8, p->stream));
        g.rb.hi = 0;
    }
    g.d_cursor = gt.n_groups + 2;                       // [2] result cursor [3] merge info
    g.d_rows_passed = (uint64_t*)(gt.n_groups + 4);     // [4..5] rows that passed the filter
    CK(p, cudaMemsetAsync(gt.n_groups, 0, 4 * GT_OCC_OFF, p->stream));
    k_table_init<<<grid_for((int64_t)cap, p->sm_count, 8), 256, 0, p->stream>>>(gt, ap, 0);
    CK(p, cudaGetLastError());
    p->stats.kernel_launches++;
    return BKGPU_OK;
}

// (the plan's device buffers go back to the allocator with every other buffer of the plan)
void agg_close(AggState& g) {
    if (g.wait_event) cudaEventDestroy(g.wait_event);
    if (g.h_pinned) cudaFreeHost(g.h_pinned);
    if (g.h_outv) cudaFreeHost(g.h_outv);
    if (g.rb.bytes) cudaFreeHost(g.rb.bytes);
    if (g.h_fused && !mapped_put(g.fused_bytes, g.h_fused)) cudaFreeHost(g.h_fused);
}

// the group count an earlier launch left in pinned memory: the 4-byte copy after a launch, or the counter block of a fused extraction
// (read without a synchronisation: a stale value only costs speed)
static void learn_groups(AggState& g) {
    if (g.h_pinned && g.h_pinned[0] > g.known_groups) g.known_groups = g.h_pinned[0];
    if (g.h_fused) { const uint32_t n = *(const volatile uint32_t*)g.h_fused; if (n > g.known_groups) g.known_groups = n; }
}

// device images of an extracted row: one per group expression, per aggregate its final value (+2 for an AVG blob)
static int agg_n_img(const AggPlan& ap) {
    int n = ap.n_group;
    for (int k = 0; k < ap.n_agg; k++) if (!ap.agg[k].hidden) n += ap.agg[k].kind == AG_AVG ? 3 : 1;
    return n;
}

// the mapped host buffer of the fused extraction, sized for the groups seen so far (at least 2048 rows); false = too many groups
// to extract this way (the table is then read back by k_extract)
static bool ensure_fused(bkgpu_plan* p, AggState& g, const Compiled& c) {
    uint32_t want = 2048;
    while (want < g.known_groups && want < (1u << 16)) want *= 2;
    if (want < g.known_groups) return false;
    if (g.h_fused && g.fused_cap >= want) return true;
    if (g.h_fused) {   // (a launch still running may write into it)
        cudaStreamSynchronize(p->stream);
        if (!mapped_put(g.fused_bytes, g.h_fused)) cudaFreeHost(g.h_fused);
        g.h_fused = g.d_fused = nullptr; g.fused_cap = 0;
    }
    const size_t bytes = 32 + (size_t)want * (size_t)agg_n_img(c.ap) * 9;
    uint8_t* h = mapped_take(bytes);
    if (!h && cudaHostAlloc((void**)&h, bytes, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return false; }
    if (cudaHostGetDevicePointer((void**)&g.d_fused, h, 0) != cudaSuccess) { cudaGetLastError(); cudaFreeHost(h); return false; }
    memset(h, 0, 32);
    g.h_fused = h; g.fused_bytes = bytes; g.fused_cap = want;
    return true;
}

// rb_build_agg: a launch appends at most one key per row and rb_build_agg aggregate, except where a probe row meets several build rows (such
// a launch can still overflow the pair buffer, and the request then fails at bkgpu_finish).  When the keys could outgrow the buffer, it is
// sorted and deduplicated first (a set does not depend on order), and the launch shrinks to the rows that fit
static int rb_room(bkgpu_plan* p, const Compiled& c, int64_t* rows) {
    RbState& rb = p->agg.rb;
    const uint64_t per = (uint64_t)c.n_rb, cap = rb.cap;
    if (rb.hi + (uint64_t)*rows * per > cap) {
        uint64_t n = 0;
        const int rc = rb_compact(p, &n);
        if (rc) return rc;
        rb.hi = n;
        const int64_t fit = (int64_t)((cap - n) / per) & ~7ll;   // (a multiple of 8 rows: the next launch's validity bitmaps stay byte-aligned)
        if (fit < 8)
            return p->fail(BKGPU_ETOOBIG, "rb_build_agg: the pair buffer holds %llu distinct (group, value) pairs and is full: raise rb_pair_capacity",
                           (unsigned long long)n);
        if (*rows > fit && !p->join.tail_launch) *rows = fit;   // (the join's tail walks every build row in one launch)
    }
    rb.hi += (uint64_t)*rows * per;
    return BKGPU_OK;
}

int launch_agg_batch(bkgpu_plan* p, AggState& g, const Compiled& c, const DevCol* cols, int64_t nrows, bool vec_ok, const JoinProbe* jp) {
    AggEnv env = g.env;   // the options, and what this launch adds to them
    env.fx_off = g.fx_off;
    env.tail_launch = p->join.tail_launch;
    // (a table that only k_apply_lookup reads is never extracted: its launches do not extract it either)
    env.multi_rank = p->nccl_comm && p->nranks > 1; env.has_post = p->c.post != nullptr || g.lookup_only;
    if (c.ap.n_keyw > 0 && env.smem_cap_log2 < 0) learn_groups(g);   // (the shared table is sized from it)
    env.known_groups = g.known_groups;
    AggArgs a; AggSelection sel;
    const int rc = select_agg_launch(c, cols, nrows, vec_ok, jp, env, a, sel);
    if (rc == BKGPU_ENOMEM) return p->fail(rc, "lean kernel: shared table does not fit");
    if (rc) return rc;
    a.gt = g.gt; a.rows_passed = g.d_rows_passed;
    if (c.kind == PK_JOIN_AGG) a.join = join_args(p, p->join.tail_launch);
    if (sel.fused_ok && ensure_fused(p, g, c)) { a.fused_out = g.d_fused; a.fused_cap = g.fused_cap; }
    const int64_t kMax = (int64_t)1 << 30;  // rows per launch (32-bit counters inside a CTA)
    int64_t algo_bytes_per_row = 0;
    for (int i = 0; i < a.n_cols; i++) algo_bytes_per_row += storage_bytes(a.cols[i].stype);
    int64_t b_rows = 0;
    for (int64_t off = 0; off < nrows; off += b_rows) {
        AggArgs b = a;
        b.nrows = std::min(kMax, nrows - off);
        if (c.n_rb) {   // (a compaction swaps the pair buffer with the sort's second buffer)
            const int rrc = rb_room(p, c, &b.nrows);
            if (rrc) return rrc;
            b.rb_keys = g.rb.keys; b.rb_ctr = g.rb.ctr; b.rb_cap = g.rb.cap;
        }
        b_rows = b.nrows;
        for (int i = 0; i < b.n_cols; i++) b.cols[i] = col_at(a.cols[i], off);
        EventPair* ep = timer_begin(p, p->timed, b.nrows * algo_bytes_per_row, false);
        cudaError_t e = launch_agg(b, sel.kernel, sel.smem, p->sm_count, p->stream, ep ? ep->a : nullptr);
        timer_end(p, ep);
        g.fused_last = b.fused_out != nullptr;
        if (e != cudaSuccess) return p->cuda_fail(e, "launch_agg");
        snprintf(p->stats.main_kernel_name, sizeof p->stats.main_kernel_name, "%s", agg_kernel_name(sel.kernel));
        p->stats.kernel_launches++;
    }
    return BKGPU_OK;
}

static int agg_batch(bkgpu_plan* p, const DevCol* cols, int64_t nrows, int64_t, bool vec_ok) { return launch_agg_batch(p, p->agg, p->c, cols, nrows, vec_ok); }

// MERGE_AGG of hll_add_agg over host memory: every non-NULL input value must be a RAW sketch, or the push fails (device-resident input is
// checked by the merge kernel itself, and the request then fails at bkgpu_finish)
static int hll_check_host_sketches(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows) {
    const AggPlan& ap = p->c.ap;
    for (int k = 0; k < ap.n_agg; k++) {
        if (ap.agg[k].kind != AG_HLL || ap.agg[k].arg_prim != BK_HLL) continue;
        const ColRef& w = p->c.cols[ap.agg[k].hll_col];
        for (int i = 0; i < ncols; i++) {
            if (cols[i].tuple_id != w.tuple_id || cols[i].slot_id != w.slot_id || !cols[i].values || cols[i].length != nrows) continue;   // (bind_columns reports those)
            for (int64_t r = 0; r < nrows; r++) {
                if (cols[i].validity && !((cols[i].validity[r >> 3] >> (r & 7)) & 1)) continue;
                const uint8_t* v = (const uint8_t*)cols[i].values + (size_t)r * HLL_RAW_BYTES;
                if (memcmp(v, "HYLL", 4) != 0 || v[4] != HLL_ENC_RAW)
                    return p->fail(BKGPU_EINVAL, "column %d_%d row %lld is not a RAW HLL sketch (\"HYLL\", encoding 255, 16400 bytes): MERGE_AGG of hll_add_agg "
                                   "merges RAW sketches only", w.tuple_id, w.slot_id, (long long)r);
            }
        }
    }
    return BKGPU_OK;
}

// a PK_AGG batch
int agg_push(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    if (p->c.sub) return apply_push(p, cols, ncols, nrows, on_device);   // (a scalar subquery: apply.cu)
    int rc = on_device ? BKGPU_OK : hll_check_host_sketches(p, cols, ncols, nrows);
    if (rc) return rc;
    rc = feed(p, p->c.cols, cols, ncols, nrows, on_device, agg_batch);
    if (rc) return rc;
    return learn_groups_async(p, p->agg, p->c);
}

// learn the cardinality for later batches' table size (no sync: a stale value only costs speed); a launch that extracted its result has
// already left the count in h_fused
int learn_groups_async(bkgpu_plan* p, AggState& g, const Compiled& c) {
    if (c.ap.n_keyw > 0 && g.env.smem_cap_log2 < 0 && g.h_pinned && !g.fused_last)
        CK(p, cudaMemcpyAsync(g.h_pinned, g.gt.n_groups, 4, cudaMemcpyDeviceToHost, p->stream));
    return BKGPU_OK;
}

// groups per rank in the exchanged partial state: never more than the group table can hold (every rank runs the same plan with
// the same options, so all ranks agree on it) — a 2^14-slot table ships 0.8 MB per rank instead of the 3 MB of the default cap
static uint32_t eff_pcap(const bkgpu_plan* p) {
    const int64_t table = p->c.ap.n_keyw == 0 ? 1 : (int64_t)1 << p->agg.group_cap_log2;
    return (uint32_t)std::min<int64_t>(p->agg.partial_cap, table);
}

// the collective step of bkgpu_finish: regions -> one set per GPU, the per-GPU partial tables meet once and are folded by K3.
// Default: compact rows, one ncclAllGather of 1 + bound x (key + lane words) per rank — `bound` = the largest group count any rank
// held in earlier runs of this plan (2048 on the first run); the merge reports the true maximum and the exchange is repeated once
// with a larger bound when it did not fit.  Option repartition: all-to-all by key owner.  Runs only with two or more ranks.
static int agg_collective(bkgpu_plan* p, bool* rows_mode) {
    const AggPlan& ap = p->c.ap;
    AggState& g = p->agg;
    GroupTable& gt = g.gt;
    *rows_mode = false;
    const uint32_t pcap = eff_pcap(p);
    int rc;
    const bool repart = g.repartition && ap.n_keyw > 0;   // (a scalar aggregate has one group: nothing to partition)
    EventPair* ep = timer_begin(p, p->timed_coll, 0);
    if (!repart) {
        *rows_mode = true;
        if (g.rank < 0 && nccl_comm_rank(p->nccl_comm, &g.rank) != 0) return p->fail(BKGPU_ENCCL, "ncclCommUserRank: %s", nccl_last_error());
        uint32_t bound = g.merge_bound ? g.merge_bound : 2048u;
        if (ap.n_keyw == 0) bound = 1;
        bound = std::min<uint32_t>(bound, pcap);
        const size_t rw = (size_t)(ap.n_keyw + ap.n_lanes + ap.n_hll * HLL_ROW_WORDS);
        const size_t words = 1 + rw * bound;
        if ((rc = ensure_buf(p, (void**)&g.d_partial, &g.d_partial_cap, words * 8))) return rc;
        if ((rc = ensure_buf(p, (void**)&g.d_gather, &g.d_gather_cap, words * 8 * (size_t)p->nranks))) return rc;
        CK(p, cudaMemsetAsync(g.d_partial, 0, 8, p->stream));
        k_partial_export_rows<<<grid_for((int64_t)gt.cap_mask + 1, p->sm_count, 1), 256, 0, p->stream>>>(gt, ap, g.d_partial, bound);
        CK(p, cudaGetLastError());
        if (nccl_all_gather(p->nccl_comm, g.d_partial, g.d_gather, words, p->stream) != 0) return p->fail(BKGPU_ENCCL, "ncclAllGather: %s", nccl_last_error());
        const int gx = (int)std::min<uint32_t>(std::max<uint32_t>((bound + 255) / 256, 1), 64);
        k_partial_merge_rows<<<dim3((unsigned)gx, (unsigned)p->nranks), 256, 0, p->stream>>>(gt, ap, g.d_gather, words, bound, p->nranks, g.rank, g.d_cursor + 1);
        CK(p, cudaGetLastError());
        g.merge_bound_used = bound;
        p->stats.kernel_launches += 2;
        timer_end(p, ep);
        return BKGPU_OK;
    }
    // hash repartition: every rank keeps only the groups it owns — an all-to-all of per-owner segments instead of the
    // all-gather; the merged table (and the result) of a rank is its partition, the union over ranks is the answer
    const size_t words = 1 + (size_t)(ap.n_keyw + ap.n_lanes) * pcap;
    if ((rc = ensure_buf(p, (void**)&g.d_partial, &g.d_partial_cap, words * 8 * (size_t)p->nranks))) return rc;
    if ((rc = ensure_buf(p, (void**)&g.d_gather, &g.d_gather_cap, words * 8 * (size_t)p->nranks))) return rc;
    if (!g.d_part_cursors && (rc = dev_alloc(p, (void**)&g.d_part_cursors, 4 * (size_t)p->nranks))) return rc;
    if (p->nranks > 1024) return p->cuda_fail(cudaErrorInvalidValue, "k_partial_counts: more than 1024 ranks");
    CK(p, cudaMemsetAsync(g.d_part_cursors, 0, sizeof(uint32_t) * (size_t)p->nranks, p->stream));
    k_partial_export_parts<<<grid_for((int64_t)gt.cap_mask + 1, p->sm_count, 8), 256, 0, p->stream>>>(gt, ap, g.d_partial, words, pcap, g.d_part_cursors, p->nranks);
    k_partial_counts<<<1, 1024, 0, p->stream>>>(g.d_partial, words, g.d_part_cursors, pcap, p->nranks);
    CK(p, cudaGetLastError());
    if (nccl_all_to_all(p->nccl_comm, g.d_partial, g.d_gather, words, p->nranks, p->stream) != 0) return p->fail(BKGPU_ENCCL, "all-to-all: %s", nccl_last_error());
    k_table_init<<<grid_for((int64_t)gt.cap_mask + 1, p->sm_count, 8), 256, 0, p->stream>>>(gt, ap, 1);   // (keeps the overflow flag an export beyond partial_capacity raised)
    CK(p, cudaGetLastError());
    k_partial_merge<<<grid_for(pcap, p->sm_count, 8), 256, 0, p->stream>>>(gt, ap, g.d_gather, words, pcap, p->nranks);
    CK(p, cudaGetLastError());
    timer_end(p, ep);
    p->stats.kernel_launches += 4;
    return BKGPU_OK;
}

// [LIMIT ->] [SORT ->] [HAVING ->] above the aggregate: the extracted rows (still on the device) become typed columns and run through
// the post fragment's sort / filter kernels; only the final rows travel to the host.  Window stages above the aggregate (post kind
// PK_WINDOW): the rows that pass HAVING are retained, then run through the stages (window.cu) and the query's ORDER BY above them.
static int agg_post(bkgpu_plan* p, uint32_t n_out, uint32_t out_cap) {
    const size_t nc = p->c.post->cols.size();
    sort_reset(p->post);
    bkgpu_stats scratch{};   // (the post fragment's kernels are not the request's "main kernel")
    int rc = sort_feed(p->post, n_out, std::max<int64_t>(n_out, 2048), 16, &scratch, [&](RowStore& in) {
        PostCols pcs; memset(&pcs, 0, sizeof pcs);
        pcs.n = (int)nc;
        int img = 0;
        for (size_t c = 0; c < nc; c++) {   // (post columns = the aggregate's output columns, in order: plan.cpp::lower_post)
            pcs.img[c] = img; pcs.stype[c] = prim_storage(in.cols[c].prim); pcs.values[c] = in.cols[c].vals; pcs.null_bytes[c] = in.cols[c].nulls;
            img += p->c.out_cols[c].kind == 1 ? 2 : 1;
        }
        k_images_to_columns<<<grid_for(n_out, p->sm_count, 8), 256, 0, p->stream>>>(p->agg.d_outv, p->agg.d_outn, out_cap, n_out, pcs);
        CK(p, cudaGetLastError());
        return BKGPU_OK;
    });
    p->stats.kernel_launches += 1 + (int64_t)nc;   // (the extraction into columns and the packs, counted with no rows too)
    if (rc) return rc;
    if (p->c.post->kind == PK_WINDOW) rc = window_finish(p, *p->c.post, p->post, p->outer, &scratch);
    else rc = sort_finish(p->post, nullptr, 1, &scratch, p->c.out_cols.data());
    if (rc) return rc;
    p->stats.kernel_launches += scratch.kernel_launches;
    return BKGPU_OK;
}

// the one wait of a request.  With several ranks on a host whose CPU budget is small (8 ranks under a 16-CPU cgroup quota: two CPUs per
// rank for the python thread, NCCL's proxy thread and this wait) a spinning wait burns the quota the other ranks' launches need:
// there the thread sleeps on a blocking-sync event instead (option blocking_sync: -1 auto, 0 spin, 1 sleep)
static int agg_wait(bkgpu_plan* p) {
    AggState& g = p->agg;
    const double t0 = HostClock::now();
    if (g.blocking_wait) {
        if (!g.wait_event) CK(p, cudaEventCreateWithFlags(&g.wait_event, cudaEventBlockingSync | cudaEventDisableTiming));
        CK(p, cudaEventRecord(g.wait_event, p->stream));
        CK(p, cudaEventSynchronize(g.wait_event));
    } else CK(p, cudaStreamSynchronize(p->stream));
    p->hclk.extract_wait += HostClock::now() - t0;
    return BKGPU_OK;
}

// what the counter block of a finished request tells the plan: rows that passed, FX's exact-path count, the groups it holds
int agg_take_counters(bkgpu_plan* p, AggState& g, const uint32_t* ctr) {
    memcpy(&g.rows_passed_host, ctr + 4, 8);
    // FX: values beyond the sampled scale are added exactly, one global atomic each; a plan whose double columns keep producing many of them
    // (a column spanning dozens of binades, outliers dominating the sample) goes back to the CAS kernel for its later launches
    if (ctr[GT_FX_EXACT] > 4096 && (uint64_t)ctr[GT_FX_EXACT] * 64 > (uint64_t)std::max<int64_t>(g.rows_passed_host, 1)) g.fx_off = 1;
    if (ctr[1]) return p->fail(BKGPU_ETOOBIG, "%s overflow (capacity 2^%d slots / partial_capacity %lld): raise group_capacity_log2",
                               g.table_name, (int)g.gt.cap_log2, (long long)g.partial_cap);
    if (ctr[0] > g.known_groups) g.known_groups = ctr[0];
    g.finish_groups = ctr[0];
    return BKGPU_OK;
}

// a BITMAP column (bkgpu.h): one bitmap per row, each the device's bytes for (slot, rb_idx), or the 8-byte empty bitmap
// ("3a300000 00000000": the reference's initialize gives every group an empty bitmap, so a group whose values were all NULL returns it)
static void rb_column(bkgpu_plan* p, HostCol& hc, const uint64_t* slot, int64_t rows, int rb_idx) {
    static const uint8_t empty[8] = {0x3a, 0x30, 0, 0, 0, 0, 0, 0};
    RbState& rb = p->agg.rb;
    std::vector<int64_t> b((size_t)rows);   // each row's bitmap in the directory, -1 = none
    int64_t total = 0;
    for (int64_t r = 0; r < rows; r++) {
        const uint32_t id = (uint32_t)(slot[r] << 2) | (uint32_t)rb_idx;
        const auto it = std::lower_bound(rb.bid.begin(), rb.bid.end(), id);
        b[r] = it != rb.bid.end() && *it == id ? (int64_t)(it - rb.bid.begin()) : -1;
        total += b[r] < 0 ? 8 : (int64_t)(rb.off[b[r] + 1] - rb.off[b[r]]);
    }
    std::vector<uint8_t>& col = rb.col[rb_idx];
    col.resize(((size_t)rows + 1) * 8 + (size_t)total);
    int64_t* offs = (int64_t*)col.data();
    uint8_t* d = col.data() + ((size_t)rows + 1) * 8;
    offs[0] = 0;
    for (int64_t r = 0; r < rows; r++) {
        const size_t len = b[r] < 0 ? 8 : (size_t)(rb.off[b[r] + 1] - rb.off[b[r]]);
        memcpy(d + offs[r], b[r] < 0 ? empty : rb.bytes + rb.off[b[r]], len);
        offs[r + 1] = offs[r] + (int64_t)len;
    }
    hc.elem = -1;
    hc.varlen = &col;
}

// typed host columns from `n_out` extracted rows (images + null bytes, column-major with stride `stride`), after OFFSET / LIMIT
static void agg_result(bkgpu_plan* p, const uint64_t* hv, const uint8_t* hn, size_t stride, uint32_t n_out) {
    const int64_t rows = n_out;
    const int64_t skip = p->c.offset > 0 ? std::min<int64_t>(p->c.offset, rows) : 0;
    int64_t lim = p->c.agg_limit;   // AggNode::get_next stops at its limit (agg_node.cpp:555)
    if (p->c.limit >= 0 && (lim < 0 || p->c.limit < lim)) lim = p->c.limit;
    int64_t keep = rows - skip;
    if (lim >= 0 && keep > lim) keep = lim;
    p->result.clear();
    int img = 0, rb_idx = 0;
    for (const OutCol& oc : p->c.out_cols) {
        HostCol hc; hc.desc = oc;
        const uint64_t* v = hv + (size_t)img * stride + skip;
        const uint8_t* nb = hn + (size_t)img * stride + skip;
        if (oc.kind == 3) {   // rb_build_agg: the group's slot, whose bitmap the device build serialized (a group without a value: the empty one)
            rb_column(p, hc, v, keep, rb_idx++);
            img++;
            p->result.push_back(std::move(hc));
            continue;
        }
        hc.elem = oc.kind == 1 ? 16 : oc.kind == 2 ? HLL_RAW_BYTES : storage_bytes(prim_storage(oc.prim));
        hc.values.assign((size_t)std::max<int64_t>(keep, 1) * (size_t)hc.elem, 0);
        // (a NULL's image is 0, which is also what a NULL row's value bytes hold)
        uint8_t* d = hc.values.data();
        if (oc.kind == 1) {
            const uint64_t* v2 = hv + (size_t)(img + 1) * stride + skip;
            for (int64_t r = 0; r < keep; r++) { memcpy(d + (size_t)r * 16, v + r, 8); memcpy(d + (size_t)r * 16 + 8, v2 + r, 8); }
        } else if (oc.kind == 2) {
            // hll_row_init's RAW sketch (hll_common.cpp:834-842): "HYLL", encoding HLL_RAW, then the registers.  hll_row_add invalidates the
            // cached cardinality (bit 7 of header byte 15) whenever a register grows, which the first value always does: a group that
            // received a value has the bit set, a group without one (every argument NULL) is the empty sketch with the byte 0
            for (int64_t r = 0; r < keep; r++) {
                uint8_t* o = d + (size_t)r * HLL_RAW_BYTES;
                memcpy(o, "HYLL", 4); o[4] = HLL_ENC_RAW;
                if (v[r]) { o[15] = 0x80; memcpy(o + HLL_HDR_BYTES, p->agg.hll_host.data() + (size_t)(v[r] - 1) * HLL_REGISTERS, HLL_REGISTERS); }
            }
        } else switch (prim_storage(oc.prim)) {
            case ST_I32: for (int64_t r = 0; r < keep; r++) { const int32_t x = (int32_t)(int64_t)v[r]; memcpy(d + (size_t)r * 4, &x, 4); } break;
            case ST_U32: for (int64_t r = 0; r < keep; r++) { const uint32_t x = (uint32_t)v[r]; memcpy(d + (size_t)r * 4, &x, 4); } break;
            case ST_F32: for (int64_t r = 0; r < keep; r++) { double x; memcpy(&x, v + r, 8); const float f = (float)x; memcpy(d + (size_t)r * 4, &f, 4); } break;
            case ST_U8: for (int64_t r = 0; r < keep; r++) d[r] = v[r] ? 1 : 0; break;
            default:
                if (hc.elem == 8) { if (keep > 0) memcpy(d, v, (size_t)keep * 8); }
                else for (int64_t r = 0; r < keep; r++) memcpy(d + (size_t)r * hc.elem, v + r, 8);
                break;
        }
        if (keep > 0 && memchr(nb, 1, (size_t)keep)) {
            hc.validity.assign((size_t)(keep + 7) / 8 + 1, 0xFF);
            for (int64_t r = 0; r < keep; r++) if (nb[r]) { hc.validity[(size_t)r >> 3] &= (uint8_t)~(1u << (r & 7)); if (oc.kind == 0) memset(d + (size_t)r * hc.elem, 0, (size_t)hc.elem); }
        }
        img += oc.kind == 1 ? 2 : 1;
        p->result.push_back(std::move(hc));
    }
    p->result_rows = keep; p->result_pos = 0;
}

// the HLL arena's counters ([0] blocks claimed, [1] a claim found the arena full, [2] a merged value was not a RAW sketch) to the host, then
// the one synchronisation (copies the caller queued before come back with it).  A claim that found the arena full fails the request, with
// the caller's message `full` (its %u: hll_group_capacity): a sketch that lost values would be wrong, not approximate
static int hll_counters(bkgpu_plan* p, uint32_t ctr[3], const char* full) {
    const GroupTable& gt = p->agg.gt;
    ctr[0] = ctr[1] = ctr[2] = 0;
    if (gt.hll_ctr) CK(p, cudaMemcpyAsync(ctr, gt.hll_ctr, 12, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    if (ctr[2]) return p->fail(BKGPU_EINVAL, "MERGE_AGG of hll_add_agg: an input value is not a RAW HLL sketch (\"HYLL\", encoding 255, 16400 bytes)");
    if (ctr[1] || ctr[0] > gt.hll_cap) return p->fail(BKGPU_ETOOBIG, full, gt.hll_cap);
    return BKGPU_OK;
}

// hll_add_agg: the arena's claimed blocks to the host (the extracted rows reference them), after the request's last kernel
static int hll_fetch(bkgpu_plan* p) {
    if (!p->c.ap.n_hll) return BKGPU_OK;
    AggState& g = p->agg;
    uint32_t ctr[3];
    int rc;
    if ((rc = hll_counters(p, ctr, "hll_add_agg: more than %u sketches (groups x hll_add_agg aggregates with a value): raise hll_group_capacity"))) return rc;
    g.hll_host.resize((size_t)ctr[0] * HLL_REGISTERS);
    if (ctr[0]) CK(p, cudaMemcpy(g.hll_host.data(), g.gt.hll_regs, (size_t)ctr[0] * HLL_REGISTERS, cudaMemcpyDeviceToHost));
    p->stats.d2h_bytes += (int64_t)g.hll_host.size() + 8;
    return BKGPU_OK;
}

// The table's groups into the pinned landing area (g.h_outv / h_outn, rows of stride g.out_cap_alloc).  The extraction is speculative, into
// the buffers kept from earlier runs: the counter block and the rows come back in ONE synchronisation; only a result larger than the buffers
// costs a second one.  ctr: the counter block ([0] groups [1] overflow [2] rows extracted [3] merge info [4..5] rows passed).
// `rows_mode`: an all-gather ran before (agg_collective); when some rank held more groups than it was sized for, nothing was merged and this
// returns after the first synchronisation, for the caller to exchange again
static int agg_extract(bkgpu_plan* p, bool rows_mode, uint32_t ctr[8]) {
    const AggPlan& ap = p->c.ap;
    AggState& g = p->agg;
    const int n_img = agg_n_img(ap);
    int rc;
    for (int attempt = 0; attempt < 2; attempt++) {
        uint32_t want = std::max<uint32_t>(std::max<uint32_t>(g.known_groups, 1), attempt ? std::max<uint32_t>(ctr[0], 1) : 1);
        if (ap.n_keyw == 0) want = 1;
        if (g.out_cap_alloc < want) {
            dev_free(p, g.d_outv); g.d_outv = nullptr; g.d_outn = nullptr;
            size_t cap = std::max<size_t>(want, 2048);
            if ((rc = dev_alloc(p, (void**)&g.d_outv, cap * 9 * (size_t)n_img + 64))) return rc;   // values, then the null bytes: ONE copy brings both back
            g.d_outn = (uint8_t*)(g.d_outv + cap * (size_t)n_img);
            g.out_cap_alloc = cap;
        }
        const uint32_t out_cap = (uint32_t)g.out_cap_alloc;
        CK(p, cudaMemsetAsync(g.d_cursor, 0, sizeof(uint32_t), p->stream));
        k_extract<<<grid_for((int64_t)g.gt.cap_mask + 1, p->sm_count, 1), 256, 0, p->stream>>>(g.gt, ap, g.d_outv, g.d_outn, out_cap, g.d_cursor, p->c.emit_default ? 1 : 0);
        CK(p, cudaGetLastError());
        p->stats.kernel_launches++;
        const size_t n_words = (size_t)out_cap * (size_t)n_img;
        if (g.h_out_cap < n_words) {   // pinned: the copies below are truly asynchronous and land in one synchronisation
            if (g.h_outv) cudaFreeHost(g.h_outv);
            g.h_outv = nullptr; g.h_outn = nullptr; g.h_out_cap = 0;
            CK(p, cudaHostAlloc((void**)&g.h_outv, n_words * 9 + 64, cudaHostAllocDefault));
            g.h_out_cap = n_words;
        }
        g.h_outn = (uint8_t*)(g.h_outv + n_words);
        // two copies, one synchronisation: the 32-byte counter block and the extracted rows (values + null bytes, contiguous on both sides)
        uint32_t local_ctr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        uint32_t* hc = g.h_pinned ? g.h_pinned + 8 : local_ctr;
        CK(p, cudaMemcpyAsync(hc, g.gt.n_groups, 32, cudaMemcpyDeviceToHost, p->stream));
        if ((const uint8_t*)g.d_outn == (const uint8_t*)(g.d_outv + n_words)) CK(p, cudaMemcpyAsync(g.h_outv, g.d_outv, n_words * 9, cudaMemcpyDeviceToHost, p->stream));
        else {
            CK(p, cudaMemcpyAsync(g.h_outv, g.d_outv, n_words * 8, cudaMemcpyDeviceToHost, p->stream));
            CK(p, cudaMemcpyAsync(g.h_outn, g.d_outn, n_words, cudaMemcpyDeviceToHost, p->stream));
        }
        if ((rc = agg_wait(p))) return rc;
        memcpy(ctr, hc, 32);
        if (rows_mode) {
            if (ctr[3] > g.merge_bound_used) return BKGPU_OK;   // nothing was merged (k_partial_merge_rows)
            const uint32_t learned = (std::max<uint32_t>(ctr[3], 1u) + 63u) & ~63u;   // the bound of the next request's all-gather
            if (learned > g.merge_bound) g.merge_bound = learned;
        }
        p->stats.d2h_bytes += (int64_t)(n_words * 9 + 12);
        if ((rc = agg_take_counters(p, p->agg, ctr))) return rc;
        if (ctr[2] <= out_cap) break;   // everything fitted
    }
    return BKGPU_OK;
}

// the result of the request from the table: `exchange` = first merge it with the other ranks' tables (agg_collective)
static int agg_finish_table(bkgpu_plan* p, bool exchange) {
    AggState& g = p->agg;
    int rc;
    // 1. the request ended with a launch that extracted its own result into mapped host memory: one wait, nothing else on the device
    if (g.fused_last && !exchange && !p->c.post) {
        if ((rc = agg_wait(p))) return rc;
        const uint32_t* ctr = (const uint32_t*)g.h_fused;
        if ((rc = agg_take_counters(p, p->agg, ctr))) return rc;
        const uint32_t n = ctr[0];
        if (n <= g.fused_cap) {
            const int n_img = agg_n_img(p->c.ap);
            p->stats.d2h_bytes += (int64_t)(32 + (size_t)n * (size_t)n_img * 9);
            const uint64_t* hv = (const uint64_t*)(g.h_fused + 32);
            agg_result(p, hv, (const uint8_t*)(hv + (size_t)n * (size_t)n_img), n, n);
            return BKGPU_OK;
        }
        // more groups than the buffer holds: the table is read back below (the next launch's buffer is sized for them)
    }
    // 2. [the exchange ->] the extraction; a round is repeated only when some rank held more groups than the all-gather was sized for
    uint32_t ctr[8];
    for (int round = 0;; round++) {
        bool rows_mode = false;
        { const double t0 = HostClock::now(); if (exchange && (rc = agg_collective(p, &rows_mode))) return rc; p->hclk.collective += HostClock::now() - t0; }
        if ((rc = agg_extract(p, rows_mode, ctr))) return rc;
        if (!rows_mode || ctr[3] <= g.merge_bound_used) break;
        if (ctr[3] > eff_pcap(p)) return p->fail(BKGPU_ETOOBIG, "a rank holds %u groups, more than partial_capacity %lld: raise partial_capacity", ctr[3], (long long)g.partial_cap);
        g.merge_bound = (ctr[3] + 63u) & ~63u;
        if (round == 2) return p->fail(BKGPU_ENCCL, "partial-state exchange did not converge");
    }
    // 3. the sketches and bitmaps the rows reference, then the post fragment or the host columns
    const uint32_t out_cap = (uint32_t)g.out_cap_alloc, n_out = std::min(ctr[2], out_cap);
    if ((rc = hll_fetch(p))) return rc;
    if (p->c.n_rb && (rc = rb_build(p))) return rc;
    if (p->c.post) return agg_post(p, n_out, out_cap);
    agg_result(p, g.h_outv, g.h_outn, out_cap, n_out);
    return BKGPU_OK;
}

int agg_finish(bkgpu_plan* p) {
    const int rc = agg_finish_table(p, p->nccl_comm && p->nranks > 1);
    if (!rc) p->stats.rows_filtered = p->stats.rows_scanned - (int64_t)p->agg.rows_passed_host;   // (came back with the counter block)
    return rc;
}

// Re-arm the table for the next request.  A finished run knows how many groups its table holds (the count came back with the result):
// clear those slots through the occupied list instead of re-initialising the whole capacity (2^20 slots = 44 MB by default)
int agg_reset(bkgpu_plan* p, AggState& g, const Compiled& c) {
    if (p->state == S_FINISHED && g.finish_groups >= 0 && c.ap.n_keyw > 0)
        k_table_clear<<<grid_for(g.finish_groups, p->sm_count, 8), 256, 0, p->stream>>>(g.gt, c.ap, (uint32_t)g.finish_groups);
    else k_table_init<<<grid_for((int64_t)g.gt.cap_mask + 1, p->sm_count, 8), 256, 0, p->stream>>>(g.gt, c.ap, 0);
    CK(p, cudaGetLastError());
    g.finish_groups = -1;
    g.fused_last = false;
    if (g.rb.ctr) { CK(p, cudaMemsetAsync(g.rb.ctr, 0, 8, p->stream)); g.rb.hi = 0; }   // (rb_build_agg: the pair buffer is empty again)
    p->stats.kernel_launches++;
    return BKGPU_OK;
}

// ---- partial state (bkgpu_partial_*): compact rows, the layout the in-library all-gather ships: [u64 groups][groups x (key words +
// lane words + HLL_ROW_WORDS per hll_add_agg)] ----
size_t agg_partial_bytes(const bkgpu_plan* p) {
    return 8 * (1 + (size_t)(p->c.ap.n_keyw + p->c.ap.n_lanes + p->c.ap.n_hll * HLL_ROW_WORDS) * (size_t)eff_pcap(p));
}
int agg_partial_export(bkgpu_plan* p, void* dev_dst) {
    const GroupTable& gt = p->agg.gt;
    CK(p, cudaMemsetAsync(dev_dst, 0, 8, p->stream));
    k_partial_export_rows<<<grid_for((int64_t)gt.cap_mask + 1, p->sm_count, 1), 256, 0, p->stream>>>(gt, p->c.ap, (uint64_t*)dev_dst, eff_pcap(p));
    CK(p, cudaGetLastError());
    p->stats.kernel_launches += 1;
    uint64_t held = 0; uint32_t ov = 0, hll_ctr[3];
    CK(p, cudaMemcpyAsync(&held, dev_dst, 8, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaMemcpyAsync(&ov, gt.overflow, 4, cudaMemcpyDeviceToHost, p->stream));
    int rc;
    if ((rc = hll_counters(p, hll_ctr, "hll_add_agg: more than %u sketches: raise hll_group_capacity"))) return rc;
    if (ov) return p->fail(BKGPU_ETOOBIG, "group table overflow (capacity 2^%d slots): raise group_capacity_log2", (int)gt.cap_log2);
    if (held > eff_pcap(p)) return p->fail(BKGPU_ETOOBIG, "this rank holds %llu groups, more than partial_capacity=%lld", (unsigned long long)held, (long long)p->agg.partial_cap);
    return BKGPU_OK;
}
// fold `nranks` exported partial states into the table, then finish the request on this plan alone
int agg_partial_merge(bkgpu_plan* p, const void* dev_src, int nranks) {
    AggState& g = p->agg;
    const uint32_t pcap = eff_pcap(p);
    k_table_init<<<grid_for((int64_t)g.gt.cap_mask + 1, p->sm_count, 8), 256, 0, p->stream>>>(g.gt, p->c.ap, 1);
    CK(p, cudaGetLastError());
    const int gx = (int)std::min<uint32_t>(std::max<uint32_t>((pcap + 255) / 256, 1), 64);
    k_partial_merge_rows<<<dim3((unsigned)gx, (unsigned)nranks), 256, 0, p->stream>>>(g.gt, p->c.ap, (const uint64_t*)dev_src, agg_partial_bytes(p) / 8, pcap, nranks,
                                                                                   -1 /* fold every segment */, g.d_cursor + 1);
    CK(p, cudaGetLastError());
    g.fused_last = false;   // (the merged table is read back by k_extract)
    p->stats.kernel_launches += 2;
    return agg_finish_table(p, false);   // (already merged)
}

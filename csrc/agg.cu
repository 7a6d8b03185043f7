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
#include "agg_kernels.cuh"
#include "interp.cuh"
#include "agg_select.h"

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
constexpr uint32_t JOIN_NO_ROW = 0xFFFFFFFFu;
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
// one output column of the joined rows: element `which` of each row-id tuple (`width` row ids: (probe, build) pairs of a two-table join,
// [fact, dim x D] of a star join) addresses `src`; JOIN_NO_ROW (the NULL-extended side) gives NULL.  dst_null may be nullptr when no
// element can be NULL
__global__ void k_join_rows_gather(DevCol src, const uint32_t* tuples, int width, int which, uint32_t n, int eb, uint8_t* dst, uint8_t* dst_null) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t r = tuples[(size_t)width * i + which];
        const bool isnull = r == JOIN_NO_ROW || elem_is_null(src, r);
        if (dst_null) dst_null[i] = isnull ? 1 : 0;
        const uint8_t* s = (const uint8_t*)src.values + (size_t)r * eb;
        uint8_t* d = dst + (size_t)i * eb;
        if (isnull) { for (int b = 0; b < eb; b++) d[b] = 0; continue; }
        switch (eb) {
            case 1: *d = *s; break;
            case 4: *(uint32_t*)d = *(const uint32_t*)s; break;
            case 8: *(uint64_t*)d = *(const uint64_t*)s; break;
            default: for (int b = 0; b < eb; b++) d[b] = s[b]; break;
        }
    }
}

// K4 build: insert (cast key image, row) of every non-NULL build row (Joiner::construct_hash_map, joiner.cpp:624-631)
__global__ void k_join_build(DevCol key, int from_prim, int cast_to, int64_t nrows, uint64_t* keys, uint32_t* rows, uint32_t cap_mask) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        if (elem_is_null(key, r)) continue;
        const uint64_t img = cast_prim(load_elem(key, r), from_prim, cast_to);
        uint32_t slot = hash_key1(img) & cap_mask;
        for (;;) {
            if (atomicCAS(rows + slot, 0xFFFFFFFFu, (uint32_t)r) == 0xFFFFFFFFu) { keys[slot] = img; break; }
            slot = (slot + 1) & cap_mask;
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
// Only `1 + bound * row words` cross NVLink; `bound` follows the group counts seen in earlier runs (api.cu).
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
cudaError_t launch_images_to_columns(const uint64_t* outv, const uint8_t* outn, uint32_t out_cap, uint32_t n, const PostCols& pc, cudaStream_t s) {
    if (!n) return cudaSuccess;
    int grid = (int)((n + 255) / 256); if (grid > 1056) grid = 1056;
    k_images_to_columns<<<grid, 256, 0, s>>>(outv, outn, out_cap, n, pc);
    return cudaGetLastError();
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

cudaError_t launch_agg(const AggArgs& a, AggKernel k, size_t smem, int sm_count, cudaStream_t s, cudaEvent_t start) {
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

// ---- FK -> PK fast path (see JoinFast in agg.h) ----
__global__ void k_join_minmax(DevCol key, int from_prim, int cast_to, int64_t nrows, uint64_t bias, uint64_t* mm) {
    uint64_t lo = ~0ull, hi = 0;
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r0 < nrows; r0 += 4 * T) {   // four independent loads in flight per thread
        uint64_t v[4]; bool ok[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t r = r0 + u * T;
            ok[u] = r < nrows && !elem_is_null(key, r);
            v[u] = ok[u] ? load_elem(key, r) : 0;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if (!ok[u]) continue;
            const uint64_t x = cast_prim(v[u], from_prim, cast_to) ^ bias;
            lo = x < lo ? x : lo; hi = x > hi ? x : hi;
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const uint64_t l2 = __shfl_xor_sync(0xFFFFFFFFu, lo, d), h2 = __shfl_xor_sync(0xFFFFFFFFu, hi, d);
        lo = l2 < lo ? l2 : lo; hi = h2 > hi ? h2 : hi;
    }
    if ((threadIdx.x & 31) == 0) { atomicMin((unsigned long long*)mm, (unsigned long long)lo); atomicMax((unsigned long long*)(mm + 1), (unsigned long long)hi); }
}
__global__ void k_join_build_fast(DevCol key, int from_prim, int cast_to, int64_t nrows, JoinFast jf, uint32_t* dense_w, uint64_t* packed_w, uint32_t* dup_flag) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        if (elem_is_null(key, r)) continue;   // a NULL key never matches
        const uint64_t img = cast_prim(load_elem(key, r), from_prim, cast_to);
        if (jf.mode == 1) {
            const uint64_t off = (img ^ jf.bias) - jf.dense_min;
            if (off >= jf.dense_size) { atomicExch(dup_flag + 2, 1u); continue; }   // outside the range learned from an earlier run of the plan: the host rebuilds
            if (atomicExch(dense_w + off, (uint32_t)r) != 0xFFFFFFFFu) atomicExch(dup_flag, 1u);
        } else {
            const uint32_t k32 = (uint32_t)img;
            const uint64_t v = ((uint64_t)k32 << 32) | (uint32_t)r;
            uint32_t slot = (k32 * 0x9E3779B1u) & jf.packed_mask;
            for (;;) {
                const uint64_t old = atomicCAS((unsigned long long*)(packed_w + slot), ~0ull, (unsigned long long)v);
                if (old == ~0ull) break;
                if ((uint32_t)(old >> 32) == k32) { atomicExch(dup_flag, 1u); break; }   // duplicate key: not a PK
                slot = (slot + 1) & jf.packed_mask;
            }
        }
    }
}
__device__ __forceinline__ uint32_t join_lookup(const JoinFast& jf, uint64_t img) {
    if (jf.mode == 1) {
        const uint64_t off = (img ^ jf.bias) - jf.dense_min;
        return off < jf.dense_size ? __ldg(jf.dense + off) : 0xFFFFFFFFu;
    }
    const uint32_t k32 = (uint32_t)img;
    uint32_t slot = (k32 * 0x9E3779B1u) & jf.packed_mask;
    for (;;) {
        const uint64_t v = __ldg((const unsigned long long*)(jf.packed + slot));
        if (v == ~0ull) return 0xFFFFFFFFu;
        if ((uint32_t)(v >> 32) == k32) return (uint32_t)v;
        slot = (slot + 1) & jf.packed_mask;
    }
}
// gather the build-side columns to probe-row alignment; four independent rows per thread keep the random
// lookups and gathers in flight together
__global__ void __launch_bounds__(256) k_join_gather(DevCol pk, int from_prim, int cast_to, int64_t nrows, JoinFast jf, GatherCols gc, uint32_t* miss_flag) {
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    bool miss = false;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; base < nrows; base += 4 * T) {
        uint32_t br[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t r = base + u * T;
            br[u] = 0xFFFFFFFEu;   // beyond the batch
            if (r < nrows) br[u] = elem_is_null(pk, r) ? 0xFFFFFFFFu : join_lookup(jf, cast_prim(load_elem(pk, r), from_prim, cast_to));
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t r = base + u * T;
            if (br[u] == 0xFFFFFFFEu) continue;
            if (br[u] == 0xFFFFFFFFu) { miss = true; continue; }
            for (int c = 0; c < gc.n; c++) {
                if (gc.elem[c] == 8) ((uint64_t*)gc.dst[c])[r] = __ldg((const unsigned long long*)gc.src[c] + br[u]);
                else if (gc.elem[c] == 4) ((uint32_t*)gc.dst[c])[r] = __ldg((const uint32_t*)gc.src[c] + br[u]);
                else gc.dst[c][r] = __ldg(gc.src[c] + br[u]);
            }
        }
    }
    if (__any_sync(0xFFFFFFFFu, miss) && (threadIdx.x & 31) == 0) atomicExch(miss_flag, 1u);
}
// K4 fused probe (JoinProbe): compose the grouped-by build attribute onto the key index built by k_join_build_fast
__global__ void k_join_compose(JoinFast jf, const uint32_t* attr_by_row, uint32_t* attr_of_key, uint64_t* packed_attr, uint32_t* bad_flag) {
    const uint64_t n = jf.mode == 1 ? jf.dense_size : (uint64_t)jf.packed_mask + 1;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (jf.mode == 1) {
            const uint32_t r = jf.dense[i];
            attr_of_key[i] = r == 0xFFFFFFFFu ? 0u : __ldg(attr_by_row + r);
        } else {
            const uint64_t e = jf.packed[i];
            uint64_t o = ~0ull;
            if (e != ~0ull) {
                o = (e & 0xFFFFFFFF00000000ull) | __ldg(attr_by_row + (uint32_t)e);
                if (o == ~0ull) atomicExch(bad_flag, 1u);   // (key, attribute) = (0xFFFFFFFF, 0xFFFFFFFF) would read as a free slot
            }
            packed_attr[i] = o;
        }
    }
}

// ---- K4 star join (PK_STAR_AGG): one fact table INNER-joined to up to four dimensions ----
// Build time: the conjuncts over one dimension alone, once per dimension row.  A row's build key is valid when the key is not NULL and the
// conjunction is TRUE: this bitmap (beside the column's own) is the key's validity for k_join_build_fast / k_join_build, which skip NULL keys.
// The two-table join runs it over a child's own filter: the build side's (with `dropped`: a row whose conjunction is not TRUE, whatever its
// key, is marked 2 in matched[]) and each probe batch's.  The program reads the row both as the probe row and as the build row.
__global__ void __launch_bounds__(256) k_star_dim_filter(const __grid_constant__ StarFilter a, uint32_t* keybits, uint8_t* dropped) {
    const int lane = threadIdx.x & 31;
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    for (int64_t w0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); w0 < a.nrows; w0 += T) {   // (warp-uniform: one bitmap word per warp and pass)
        const int64_t r = w0 + lane;
        bool ok = r < a.nrows && !elem_is_null(a.cols[a.key_col], r);
        if ((ok || (dropped && r < a.nrows)) && a.prog.n_instr > 0) {
            uint64_t out[1]; uint32_t out_null;
            run_program(a.prog, a.cols, r, out, out_null, r);
            const bool pass = !(out_null & 1u) && out[0] != 0;
            ok = ok && pass;
            if (dropped && !pass) dropped[r] = 2;
        }
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, ok);
        if (lane == 0) keybits[w0 >> 5] = m;
    }
}
// four consecutive foreign keys [r0, r0 + 4) as canonical images: one 128-bit load (4-byte keys) or two (8-byte keys) when the chunk is 32-byte
// aligned and the four rows exist
__device__ __forceinline__ void load_quad(const DevCol& c, int64_t r0, int64_t nrows, bool vec, uint64_t (&v)[4]) {
    if (vec && r0 + 4 <= nrows && (c.stype == ST_I32 || c.stype == ST_U32)) {
        const uint4 q = __ldg((const uint4*)((const uint32_t*)c.values + r0));
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int u = 0; u < 4; u++) v[u] = narrow_prim(c.stype == ST_I32 ? (uint64_t)(int64_t)(int32_t)w[u] : (uint64_t)w[u], c.prim);
        return;
    }
    if (vec && r0 + 4 <= nrows && (c.stype == ST_I64 || c.stype == ST_U64)) {
        const ulonglong2 a = __ldg((const ulonglong2*)((const unsigned long long*)c.values + r0));
        const ulonglong2 b = __ldg((const ulonglong2*)((const unsigned long long*)c.values + r0 + 2));
        v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
        return;
    }
#pragma unroll
    for (int u = 0; u < 4; u++) v[u] = r0 + u < nrows ? load_elem(c, r0 + u) : 0;
}
// Probe: one pass over a chunk's fact rows.  A row survives when every dimension with unique keys has a partner (a NULL foreign key has none:
// one L2-resident index read per dimension).  Survivors leave as row-id tuples [fact row, dim row x D] in any order, compacted with warp
// ballots and one cursor atomic per warp; the slots of dimensions with duplicate keys are filled by k_star_expand.
__global__ void __launch_bounds__(256) k_star_probe(const __grid_constant__ StarProbe a, uint32_t* out, uint32_t* cursor) {
    const int lane = threadIdx.x & 31;
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    const int64_t nq = (a.nrows + 3) / 4;
    for (int64_t q0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); q0 < nq; q0 += T) {   // (warp-uniform trip count: the ballots below)
        const int64_t r0 = (q0 + lane) * 4;
        uint32_t br[4][4];
        // every lookup is issued before any result is tested: up to 16 independent index reads in flight per thread
#pragma unroll
        for (int d = 0; d < 4; d++) {
            if (d >= a.n) break;
            const StarLookup& L = a.d[d];
            uint64_t v[4];
            load_quad(L.fk, r0, a.nrows, a.vec != 0, v);
#pragma unroll
            for (int u = 0; u < 4; u++)
                br[u][d] = r0 + u < a.nrows && !elem_is_null(L.fk, r0 + u) ? join_lookup(L.jf, cast_prim(v[u], L.from_prim, L.cast_prim)) : JOIN_NO_ROW;
        }
        uint32_t live = 0;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            bool ok = r0 + u < a.nrows;
#pragma unroll
            for (int d = 0; d < 4; d++) if (d < a.n) ok = ok && br[u][d] != JOIN_NO_ROW;
            if (ok) live |= 1u << u;
        }
        uint32_t b[4]; uint32_t total = 0;
#pragma unroll
        for (int u = 0; u < 4; u++) { b[u] = __ballot_sync(0xFFFFFFFFu, (live >> u) & 1u); total += (uint32_t)__popc(b[u]); }
        if (total == 0) continue;
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(cursor, total);
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if ((live >> u) & 1u) {
                uint32_t* t = out + (size_t)a.width * (base + (uint32_t)__popc(b[u] & lt));
                t[0] = (uint32_t)(r0 + u);
#pragma unroll
                for (int d = 0; d < 4; d++) if (d < a.n) t[a.d[d].slot] = br[u][d];
            }
            base += (uint32_t)__popc(b[u]);
        }
    }
}
// A dimension with duplicate keys: every tuple becomes one tuple per matching row of the dimension's multimap (k_join_build), or none.
// Past `cap` only the count goes on: the host grows the buffer to the count and runs the pass again.
__global__ void __launch_bounds__(256) k_star_expand(DevCol fk, int from_prim, int cast_to, const uint64_t* keys, const uint32_t* rows, uint32_t cap_mask,
                                                     const uint32_t* in, uint32_t n_in, int width, int slot, uint32_t* out, uint32_t cap, uint32_t* cursor) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_in; i += gridDim.x * blockDim.x) {
        const uint32_t* t = in + (size_t)width * i;
        const uint32_t f = t[0];
        if (elem_is_null(fk, f)) continue;
        const uint64_t img = cast_prim(load_elem(fk, f), from_prim, cast_to);
        for (uint32_t h = hash_key1(img) & cap_mask;; h = (h + 1) & cap_mask) {
            const uint32_t br = rows[h];
            if (br == 0xFFFFFFFFu) break;
            if (keys[h] != img) continue;
            const uint32_t pos = atomicAdd(cursor, 1u);
            if (pos >= cap) continue;
            uint32_t* o = out + (size_t)width * pos;
            for (int k = 0; k < width; k++) o[k] = t[k];
            o[slot] = br;
        }
    }
}
cudaError_t launch_star_dim_filter(const StarFilter& f, uint32_t* keybits, uint8_t* dropped, cudaStream_t s) {
    if (f.nrows == 0) return cudaSuccess;
    int grid = (int)((f.nrows + 255) / 256); if (grid > 132 * 16) grid = 132 * 16;
    k_star_dim_filter<<<grid, 256, 0, s>>>(f, keybits, dropped);
    return cudaGetLastError();
}
cudaError_t launch_star_probe(const StarProbe& sp, uint32_t* out, uint32_t* cursor, int sm_count, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(cursor, 0, 4, s);
    if (e != cudaSuccess || sp.nrows == 0) return e;
    int64_t g = (sp.nrows + 1023) / 1024; if (g > (int64_t)sm_count * 8) g = (int64_t)sm_count * 8;
    k_star_probe<<<(int)(g < 1 ? 1 : g), 256, 0, s>>>(sp, out, cursor);
    return cudaGetLastError();
}
cudaError_t launch_star_expand(const DevCol& fk, int from_prim, int cast_prim_, const uint64_t* keys, const uint32_t* rows, uint32_t cap_mask, const uint32_t* in, uint32_t n_in,
                               int width, int slot, uint32_t* out, uint32_t cap, uint32_t* cursor, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(cursor, 0, 4, s);
    if (e != cudaSuccess || n_in == 0) return e;
    int grid = (int)((n_in + 255) / 256); if (grid > 132 * 16) grid = 132 * 16;
    k_star_expand<<<grid, 256, 0, s>>>(fk, from_prim, cast_prim_, keys, rows, cap_mask, in, n_in, width, slot, out, cap, cursor);
    return cudaGetLastError();
}

cudaError_t launch_join_compose(const JoinFast& jf, const uint32_t* attr_by_row, uint32_t* attr_of_key, uint64_t* packed_attr, uint32_t* bad_flag, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(bad_flag, 0, 4, s);
    if (e != cudaSuccess) return e;
    const uint64_t n = jf.mode == 1 ? jf.dense_size : (uint64_t)jf.packed_mask + 1;
    int grid = (int)((n + 255) / 256); if (grid > 132 * 16) grid = 132 * 16; if (grid < 1) grid = 1;
    k_join_compose<<<grid, 256, 0, s>>>(jf, attr_by_row, attr_of_key, packed_attr, bad_flag);
    return cudaGetLastError();
}
cudaError_t launch_join_minmax(const DevCol& key, int from_prim, int cast_prim_, int64_t nrows, uint64_t bias, uint64_t* mm, cudaStream_t s) {
    const uint64_t init[2] = {~0ull, 0ull};
    cudaError_t e = cudaMemcpyAsync(mm, init, 16, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess || nrows == 0) return e;
    int grid = (int)((nrows + 255) / 256); if (grid > 132 * 8) grid = 132 * 8;
    k_join_minmax<<<grid, 256, 0, s>>>(key, from_prim, cast_prim_, nrows, bias, mm);
    return cudaGetLastError();
}
cudaError_t launch_join_build_fast(const DevCol& key, int from_prim, int cast_prim_, int64_t nrows, const JoinFast& jf, uint32_t* dense_w, uint64_t* packed_w, uint32_t* dup_flag, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(dup_flag, 0, 12, s);   // [0] duplicate key, [1] fused probe unusable (set by the compose step), [2] key outside the guessed range
    if (e != cudaSuccess) return e;
    if (jf.mode == 1) e = cudaMemsetAsync(dense_w, 0xFF, jf.dense_size * 4, s); else e = cudaMemsetAsync(packed_w, 0xFF, ((size_t)jf.packed_mask + 1) * 8, s);
    if (e != cudaSuccess || nrows == 0) return e;
    int grid = (int)((nrows + 255) / 256); if (grid > 132 * 16) grid = 132 * 16;
    k_join_build_fast<<<grid, 256, 0, s>>>(key, from_prim, cast_prim_, nrows, jf, dense_w, packed_w, dup_flag);
    return cudaGetLastError();
}
cudaError_t launch_join_gather(const DevCol& probe_key, int from_prim, int cast_prim_, int64_t nrows, const JoinFast& jf, const GatherCols& gc, uint32_t* miss_flag, cudaStream_t s) {
    if (nrows == 0) return cudaSuccess;
    int grid = (int)((nrows + 1023) / 1024); if (grid > 132 * 8) grid = 132 * 8; if (grid < 1) grid = 1;
    k_join_gather<<<grid, 256, 0, s>>>(probe_key, from_prim, cast_prim_, nrows, jf, gc, miss_flag);
    return cudaGetLastError();
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
cudaError_t launch_join_rows_gather(const DevCol& src, const uint32_t* tuples, int width, int which, uint32_t n, int eb, uint8_t* dst, uint8_t* dst_null, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    int grid = (int)((n + 255) / 256); if (grid > 132 * 16) grid = 132 * 16;
    k_join_rows_gather<<<grid, 256, 0, s>>>(src, tuples, width, which, n, eb, dst, dst_null);
    return cudaGetLastError();
}
cudaError_t launch_join_build(const DevCol& key, int from_prim, int cast_prim_, int64_t nrows, uint64_t* keys, uint32_t* rows, uint32_t cap_mask, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(rows, 0xFF, (size_t)(cap_mask + 1) * 4, s);
    if (e != cudaSuccess || nrows == 0) return e;
    int grid = (int)((nrows + 255) / 256); if (grid > 132 * 16) grid = 132 * 16;
    k_join_build<<<grid, 256, 0, s>>>(key, from_prim, cast_prim_, nrows, keys, rows, cap_mask);
    return cudaGetLastError();
}
cudaError_t launch_table_init(const GroupTable& gt, const AggPlan& ap, cudaStream_t s, int keep_overflow) {
    const uint32_t cap = gt.cap_mask + 1;
    int grid = (int)((cap + 255) / 256); if (grid > 1056) grid = 1056;
    k_table_init<<<grid, 256, 0, s>>>(gt, ap, keep_overflow);
    return cudaGetLastError();
}
cudaError_t launch_table_clear(const GroupTable& gt, const AggPlan& ap, uint32_t n_occupied, cudaStream_t s) {
    int grid = (int)((n_occupied + 255) / 256); if (grid > 1056) grid = 1056; if (grid < 1) grid = 1;
    k_table_clear<<<grid, 256, 0, s>>>(gt, ap, n_occupied);
    return cudaGetLastError();
}
cudaError_t launch_partial_export_rows(const GroupTable& gt, const AggPlan& ap, uint64_t* dst, uint32_t bound, cudaStream_t s) {
    const uint32_t cap = gt.cap_mask + 1;
    int grid = (int)((cap + 255) / 256); if (grid > 132) grid = 132;   // (the kernel walks the occupied list, grid-stride)
    cudaError_t e = cudaMemsetAsync(dst, 0, 8, s);
    if (e != cudaSuccess) return e;
    k_partial_export_rows<<<grid, 256, 0, s>>>(gt, ap, dst, bound);
    return cudaGetLastError();
}
cudaError_t launch_partial_merge_rows(const GroupTable& gt, const AggPlan& ap, const uint64_t* src, size_t words_per_rank, uint32_t bound, int nranks, int self,
                                      uint32_t* max_count, cudaStream_t s) {
    int gx = (int)((bound + 255) / 256); if (gx > 64) gx = 64; if (gx < 1) gx = 1;
    k_partial_merge_rows<<<dim3((unsigned)gx, (unsigned)nranks), 256, 0, s>>>(gt, ap, src, words_per_rank, bound, nranks, self, max_count);
    return cudaGetLastError();
}
cudaError_t launch_partial_export_parts(const GroupTable& gt, const AggPlan& ap, uint64_t* dst, size_t words_per_seg, uint32_t pcap, uint32_t* cursors, int nranks, cudaStream_t s) {
    if (nranks > 1024) return cudaErrorInvalidValue;
    const uint32_t cap = gt.cap_mask + 1;
    int grid = (int)((cap + 255) / 256); if (grid > 1056) grid = 1056;
    cudaError_t e = cudaMemsetAsync(cursors, 0, sizeof(uint32_t) * (size_t)nranks, s);
    if (e != cudaSuccess) return e;
    k_partial_export_parts<<<grid, 256, 0, s>>>(gt, ap, dst, words_per_seg, pcap, cursors, nranks);
    k_partial_counts<<<1, 1024, 0, s>>>(dst, words_per_seg, cursors, pcap, nranks);
    return cudaGetLastError();
}
cudaError_t launch_partial_merge(const GroupTable& gt, const AggPlan& ap, const uint64_t* src, size_t words_per_rank, uint32_t pcap, int nranks, cudaStream_t s) {
    int grid = (int)((pcap + 255) / 256); if (grid > 1056) grid = 1056; if (grid < 1) grid = 1;
    k_partial_merge<<<grid, 256, 0, s>>>(gt, ap, src, words_per_rank, pcap, nranks);
    return cudaGetLastError();
}
cudaError_t launch_extract(const GroupTable& gt, const AggPlan& ap, uint64_t* outv, uint8_t* outn, uint32_t out_cap, uint32_t* cursor, int emit_default, cudaStream_t s) {
    const uint32_t cap = gt.cap_mask + 1;
    int grid = (int)((cap + 255) / 256); if (grid > 132) grid = 132;   // (the kernel walks the occupied list, grid-stride)
    cudaError_t e = cudaMemsetAsync(cursor, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    k_extract<<<grid, 256, 0, s>>>(gt, ap, outv, outn, out_cap, cursor, emit_default);
    return cudaGetLastError();
}

}  // namespace bk

// agg_kernels.cuh — device pieces shared by the aggregate kernels: row accumulation into a table slot,
// group merge (K3), shared-table carve-up and flush (see agg.cu for the overview).
#pragma once
#include "agg.h"
#include "dev_common.cuh"
#include "hll.cuh"

namespace bk {

// ------------------------------------------------------------------------------------------
// accumulate one row into a table slot (shared or global)
//
// Shared tables hold only the lanes that need per-row work in THIS batch (args.smem_lane maps a
// global lane to its shared lane or 0xFF): the non-NULL counter of an aggregate whose argument
// cannot be NULL in this batch always equals the group's row count, so it is not touched per row;
// the flush adds the shared row count to it (args.alias_mask).
// ------------------------------------------------------------------------------------------
template <bool SHARED, class ArgFn>
__device__ __forceinline__ void accumulate_row(const AggArgs& args, uint64_t* lanes, uint32_t cap, int slot, ArgFn arg) {
    const AggPlan& ap = args.plan;
    lane_atomic<SHARED>(LN_ADD_I64, lanes + slot, 1ull);  // lane 0: group row count
#pragma unroll 1
    for (int i = 0; i < ap.n_agg; i++) {
        const AggSpec a = ap.agg[i];
        if (a.kind == AG_COUNT_STAR) continue;
        uint64_t v; bool isnull;
        arg(i, v, isnull);
        if (isnull) continue;
        if (a.cnt_lane && a.cnt_owner && (!SHARED || a.nullable)) {
            const int l = SHARED ? args.smem_lane[a.cnt_lane] : a.cnt_lane;
            lane_atomic<SHARED>(LN_ADD_I64, lanes + (size_t)l * cap + slot, 1ull);
        }
        if (a.kind == AG_COUNT || !a.acc_owner) continue;
        v = to_lane_class(v, a.arg_vclass, a.vclass);
        const int l = SHARED ? args.smem_lane[a.acc_lane] : a.acc_lane;
        lane_atomic<SHARED>(ap.lane_op[a.acc_lane], lanes + (size_t)l * cap + slot, v);
    }
}

// merge the lane values of one group (a shared-table slot or an imported partial) into the global
// table: AggFnCall::merge (src/expr/agg_fn_call.cpp:779-822) lane by lane.  lane_val(l, v) yields
// the value for global lane l or returns false when the source has nothing for it.
// (a sketch lane, LN_HLL, has nothing to add here: the caller's lane_val skips it, and the sketch's registers travel apart)
template <class LaneVal>
__device__ __forceinline__ void merge_group(const AggPlan& ap, const GroupTable& gt, const uint64_t* key, LaneVal lane_val) {
    int slot = 0;
    if (ap.n_keyw > 0) {
        slot = table_upsert<false, 0>(gt.state, gt.keys, gt.cap_mask, key, ap.n_keyw,
                                      ap.n_keyw == 1 ? hash_key1(key[0]) : hash_key(key, ap.n_keyw),
                                      (int)(gt.cap_mask + 1), gt.n_groups);
        if (slot < 0) { atomicExch(gt.overflow, 1u); return; }
    }
    const uint32_t cap = gt.cap_mask + 1;
#pragma unroll 1
    for (int l = 0; l < ap.n_lanes; l++) {
        uint64_t v;
        if (!lane_val(l, v)) continue;
        const int op = ap.lane_op[l];
        if (v == lane_identity(op)) continue;
        lane_atomic<false>(op, gt.lanes + (size_t)l * cap + slot, v);
    }
}

// ------------------------------------------------------------------------------------------
// hll_add_agg (AG_HLL): a group's sketch is a 16384-byte block of the register arena, referenced by its lane as block + 1
// ------------------------------------------------------------------------------------------
// the registers of the sketch behind `lane`, claimed on first use: the first thread to CAS the lane from 0 takes the next block, zeroes it
// and publishes it; others wait for the publication.  nullptr when the arena is full (hll_ctr[1] is then set and the request fails).
static __device__ __noinline__ uint8_t* hll_sketch(const GroupTable& gt, uint64_t* lane) {
    unsigned long long v = __ldcg((const unsigned long long*)lane);
    if (v == 0) {
        v = atomicCAS((unsigned long long*)lane, 0ull, (unsigned long long)HLL_LANE_BUSY);
        if (v == 0) {
            const uint32_t b = atomicAdd(gt.hll_ctr, 1u);
            if (b >= gt.hll_cap) { atomicExch(gt.hll_ctr + 1, 1u); atomicExch((unsigned long long*)lane, (unsigned long long)HLL_LANE_FULL); return nullptr; }
            uint4* r = (uint4*)(gt.hll_regs + (size_t)b * HLL_REGISTERS);
            for (int i = 0; i < HLL_REGISTERS / 16; i++) __stcg(r + i, make_uint4(0u, 0u, 0u, 0u));
            __threadfence();   // (the zeroed block before its reference)
            atomicExch((unsigned long long*)lane, (unsigned long long)b + 1ull);
            return (uint8_t*)r;
        }
    }
    while (v == HLL_LANE_BUSY) { __nanosleep(64); v = __ldcg((const unsigned long long*)lane); }
    if (v == HLL_LANE_FULL) return nullptr;
    __threadfence();
    return gt.hll_regs + (size_t)(v - 1) * HLL_REGISTERS;
}
// register = max(register, count) on the 32-bit word holding it.  The register is read first: once a sketch has filled up, almost
// every row finds its register already as large and writes nothing.  Registers live in L2 (atomics and ld.cg), never in L1.
__device__ __forceinline__ void hll_max_word(unsigned int* w, unsigned int want, unsigned int cur) {
    for (;;) {
        const unsigned int nv = __vmaxu4(cur, want);
        if (nv == cur) return;
        const unsigned int prev = atomicCAS(w, cur, nv);
        if (prev == cur) return;
        cur = prev;
    }
}
__device__ __forceinline__ void hll_max_register(uint8_t* regs, uint32_t reg, uint32_t count) {
    unsigned int* w = (unsigned int*)(regs + (reg & ~3u));
    const uint32_t shift = (reg & 3u) * 8u;
    const unsigned int cur = __ldcg(w);
    if (((cur >> shift) & 0xFFu) < count) hll_max_word(w, count << shift, cur);
}
// MERGE_AGG: the RAW sketch at row `row` of column `c` into the sketch of `slot` (hll_merge_agg, hll_common.cpp:630-703): register-wise
// max.  The group's sketch is claimed even when no register grows, as hll_merge_agg invalidates the cached cardinality whatever it merges.
// A value whose magic or encoding is not RAW's sets hll_ctr[2] and the request fails (DENSE and SPARSE sketches vary in length)
__device__ __forceinline__ void hll_merge_value(const GroupTable& gt, const AggSpec& a, const DevCol& c, int64_t row, uint64_t* lanes, uint32_t cap, int slot) {
    const uint8_t* v = (const uint8_t*)c.values + (size_t)row * HLL_RAW_BYTES;
    const uint32_t magic = __ldg((const uint32_t*)v), enc = __ldg(v + 4);
    if (magic != 0x4C4C5948u /* "HYLL" */ || enc != HLL_ENC_RAW) { atomicExch(gt.hll_ctr + 2, 1u); return; }
    uint8_t* regs = hll_sketch(gt, lanes + (size_t)a.acc_lane * cap + slot);
    if (!regs) return;
    const uint32_t* src = (const uint32_t*)(v + HLL_HDR_BYTES);   // (16400 and 16 are multiples of 16: every value is word-aligned)
    unsigned int* dst = (unsigned int*)regs;
    for (int w = 0; w < HLL_REGISTERS / 4; w++) {
        const unsigned int x = __ldg(src + w);
        if (!x) continue;
        const unsigned int cur = __ldcg(dst + w);
        if (__vmaxu4(cur, x) != cur) hll_max_word(dst + w, x, cur);
    }
}
// one non-NULL argument value of an AG_HLL aggregate into the sketch of `slot`
__device__ __forceinline__ void hll_add_value(const GroupTable& gt, const AggSpec& a, uint64_t* lanes, uint32_t cap, int slot, uint64_t v) {
    if (a.arg_prim == BK_FLOAT && a.arg_vclass == VC_F64) v = __float_as_uint((float)bits_f64(v));   // (a computed FLOAT value: its float bytes)
    uint32_t reg;
    const int count = hll_pat_len(hll_hash(v, hll_key_bytes(a.arg_prim)), &reg);
    uint8_t* regs = hll_sketch(gt, lanes + (size_t)a.acc_lane * cap + slot);
    if (regs) hll_max_register(regs, reg, (uint32_t)count);
}

// ------------------------------------------------------------------------------------------
// shared-memory table carve-up: [keys n_keyw x cap][lanes n_smem_lanes x cap][state cap]
// ------------------------------------------------------------------------------------------
constexpr uint64_t EMPTY_KEY = 0xFFFFFFFFFFFFFFFFull;  // "free slot" marker of sentinel-mode shared tables (one-word keys)

// word index of shared lane `sl` of `slot`: SoA, or 16-byte pairs so that two lanes of a group sit in one
// 128-bit word (updated together by one ATOMS.CAS.128 in the lean kernel)
__device__ __forceinline__ size_t smem_lane_word(const AggArgs& a, int sl, uint32_t slot, uint32_t cap) {
    return a.smem_paired ? (((size_t)(sl >> 1) * cap + slot) * 2 + (size_t)(sl & 1)) : ((size_t)sl * cap + slot);
}

struct SmemTable {
    uint32_t* state; uint64_t* keys; uint64_t* lanes; uint32_t cap_mask;
};
__device__ __forceinline__ SmemTable smem_table_init(unsigned char* raw, const AggArgs& args) {
    const AggPlan& ap = args.plan;
    SmemTable t;
    const uint32_t cap = 1u << args.smem_cap_log2;
    t.cap_mask = cap - 1;
    t.keys = (uint64_t*)raw;
    t.lanes = t.keys + (size_t)args.smem_keyw * cap;
    t.state = (uint32_t*)(t.lanes + (size_t)args.n_smem_lanes * cap);
    if (args.smem_sentinel) { for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) t.keys[i] = EMPTY_KEY; }
    else { for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) t.state[i] = 0u; }
    for (int l = 0; l < ap.n_lanes; l++) {
        const int sl = args.smem_lane[l];
        if (sl == 0xFF) continue;
        const uint64_t id = lane_identity(ap.lane_op[l]);
        for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) t.lanes[smem_lane_word(args, sl, i, cap)] = id;
    }
    __syncthreads();
    return t;
}
__device__ __forceinline__ void smem_table_flush(const SmemTable& t, const AggArgs& args) {
    __syncthreads();
    const AggPlan& ap = args.plan;
    const uint32_t cap = t.cap_mask + 1;
    for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) {
        if (args.smem_sentinel ? (t.keys[i] == EMPTY_KEY) : (t.state[i] != 2u)) continue;
        uint64_t key[MAX_KEYW];
        for (int w = 0; w < ap.n_keyw; w++) key[w] = w < args.smem_keyw ? t.keys[(size_t)w * cap + i] : 0ull;  // sentinel mode: further words are 0
        merge_group(ap, args.gt, key, [&](int l, uint64_t& v) {
            const int sl = args.smem_lane[l];
            if (sl != 0xFF) { v = t.lanes[smem_lane_word(args, sl, i, cap)]; return true; }
            if ((args.alias_mask >> l) & 1u) { v = t.lanes[smem_lane_word(args, 0, i, cap)]; return true; }  // counter that follows the row count
            return false;
        });
    }
}

// ------------------------------------------------------------------------------------------
// result extraction: one output row per group.  Output columns (canonical 64-bit images + one null
// byte each, column-major with stride `stride`), in this order: group expressions, then per aggregate
// its final value and, for AVG, the intermediate {sum, count} pair (AggFnCall::finalize,
// agg_fn_call.cpp:927-990).  Reads go to L2 (ld.cg): the fused caller runs in the launch that updated the table.  Every key word
// and lane of the slot is loaded before the first store, so a group costs one round trip to L2, not one per output column.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void extract_group(const GroupTable& gt, const AggPlan& ap, uint32_t i, uint32_t pos, uint64_t* outv, uint8_t* outn, uint32_t stride) {
    const uint32_t cap = gt.cap_mask + 1;
    uint64_t kw[MAX_KEYW], lw[MAX_LANES];
#pragma unroll 4
    for (int w = 0; w < ap.n_keyw; w++) kw[w] = __ldcg((const unsigned long long*)gt.keys + (size_t)w * cap + i);
#pragma unroll 4
    for (int l = 0; l < ap.n_lanes; l++) lw[l] = __ldcg((const unsigned long long*)gt.lanes + (size_t)l * cap + i);
    const uint64_t nrows = lw[0];
    int c = 0;
    for (int g = 0; g < ap.n_group; g++, c++) {
        const bool isnull = ap.key_null_word[g] != 0xFF && ((kw[ap.key_null_word[g]] >> ap.key_null_shift[g]) & 1ull);
        uint64_t v = kw[ap.key_word[g]] >> ap.key_shift[g];
        if (ap.key_bits[g] < 64) v &= (1ull << ap.key_bits[g]) - 1ull;
        // sign-extend narrow signed keys back to their canonical image
        if (ap.key_bits[g] == 32 && prim_class(ap.key_prim[g]) == VC_I64) v = (uint64_t)(int64_t)(int32_t)v;
        outv[(size_t)c * stride + pos] = isnull ? 0 : v;
        outn[(size_t)c * stride + pos] = isnull ? 1 : 0;
    }
    for (int k = 0; k < ap.n_agg; k++) {
        const AggSpec a = ap.agg[k];
        if (a.hidden) continue;
        const uint64_t cnt = a.cnt_lane < ap.n_lanes ? lw[a.cnt_lane] : 0;   // (lane 0 = the group's row count)
        const uint64_t acc = a.acc_lane < ap.n_lanes ? lw[a.acc_lane] : 0;
        uint64_t v = 0; uint8_t isnull = 0;
        switch (a.kind) {
            case AG_COUNT_STAR: v = nrows; break;
            case AG_COUNT: v = cnt; break;
            case AG_COUNT_MERGE: case AG_HLL: v = acc; break;   // (AG_HLL: the sketch reference; the host copies its registers)
            case AG_RB: v = i; break;   // the group's slot: the host finds its bitmaps by (slot, rb_idx)
            case AG_AVG:   // (AVG's sum starts from +0.0 in the reference, agg_initialize: + 0.0 turns the lane's -0.0 into +0.0)
                if (cnt == 0) isnull = 1; else v = f64_bits(__ddiv_rn(__dadd_rn(bits_f64(acc), 0.0), (double)(int64_t)cnt));
                break;
            default: if (cnt == 0) isnull = 1; else v = acc; break;  // SUM / MIN / MAX: NULL without input
        }
        outv[(size_t)c * stride + pos] = v; outn[(size_t)c * stride + pos] = isnull; c++;
        if (a.kind == AG_AVG) {  // intermediate blob {double sum; int64 count}
            // the blank row of an empty scalar aggregate initialises only its counts (agg_node.cpp:489-503): blob stays NULL
            outv[(size_t)c * stride + pos] = f64_bits(__dadd_rn(bits_f64(acc), 0.0)); outn[(size_t)c * stride + pos] = (ap.n_keyw == 0 && nrows == 0) ? 1 : 0; c++;
            outv[(size_t)c * stride + pos] = cnt; outn[(size_t)c * stride + pos] = 0; c++;
        }
    }
}

// The end of a grouped launch that extracts its own result (AggArgs::fused_out): every CTA takes a ticket once its table updates are
// done; the CTA that draws the last one sees the whole table and writes the counter block and every group's row straight into the
// mapped host buffer, so the request needs no extraction kernel and no copies after it.  Each launch of a multi-batch request
// overwrites the previous launch's rows; the host reads them only after the last.  The table itself is left as it is (it stays the
// request's partial state until bkgpu_reset clears it).
__device__ __forceinline__ void fused_extract(const AggArgs& a) {
    __shared__ uint32_t is_last;
    __threadfence();   // this thread's table updates, before the CTA's ticket
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicAdd(a.gt.n_groups + GT_TICKET, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    const GroupTable& gt = a.gt;
    const AggPlan& ap = a.plan;
    const uint32_t n = __ldcg(gt.n_groups);
    uint32_t* ctr = (uint32_t*)a.fused_out;
    if (threadIdx.x < GT_OCC_OFF) ctr[threadIdx.x] = threadIdx.x == GT_TICKET ? 0u : __ldcg(gt.n_groups + threadIdx.x);
    if (threadIdx.x == 0) gt.n_groups[GT_TICKET] = 0u;   // (every CTA has drawn: the next launch of the request starts from 0)
    if (n > a.fused_cap) return;
    int n_img = ap.n_group;
    for (int k = 0; k < ap.n_agg; k++) if (!ap.agg[k].hidden) n_img += ap.agg[k].kind == AG_AVG ? 3 : 1;
    uint64_t* outv = (uint64_t*)(a.fused_out + 32);
    uint8_t* outn = (uint8_t*)(outv + (size_t)n_img * n);
    for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) extract_group(gt, ap, __ldcg(gt.n_groups + GT_OCC_OFF + j), j, outv, outn, n);
}


}  // namespace bk

// agg_wp.cuh — K1+K2 for the lean shape WITHOUT shared-memory atomics: warp-private accumulator tables.
//
// Why: the round-1 lean kernel (k_agg_group_lean, agg_direct.cuh) keeps ONE table per CTA and updates it with
// ATOMS (RED.u32 for the row count, an LDS.128 -> 2xDADD -> ATOMS.CAS.128 loop for the two double sums).  Spread-address
// shared atomics retire lane by lane, so two atomics per surviving row bound the kernel by the shared-memory pipe rather
// than by HBM whatever else is tuned.  Here no accumulator is ever shared
// between warps, so every update is a plain LDS / STS read-modify-write:
//
//   * key table (one per CTA, read-mostly): 16-byte buckets of two {key32 | id32 << 32} words mapping a GROUP BY key to a
//     dense group id; one LDS.128 answers a probe.  A key is inserted once per CTA (CAS on an EMPTY word, id from a shared
//     counter).  DENSE instantiation: keys known (from earlier batches / runs of the plan) to lie in a small range skip
//     the table, id = key - range start.
//   * accumulators (one set per WARP, indexed by the dense id): cnt[id] (u32) and sums[id] (8 bytes per value column;
//     two columns share a 16-byte word moved by LDS.128 / STS.128).
//   * no compaction queue: every lane keeps its four rows in registers; four predicates guard the four "entry slots".
//   * lanes of one warp that hit the same id in the same round are arbitrated through the count word itself: every
//     pending entry reads cnt, all write (cnt + 1) with their tag (entry slot * 32 + lane) in the low 7 bits, all read
//     back; the entry whose word survived owns the group for this round and adds its values, the others go round again
//     (1000 groups, 64 entries: ~2 entries lose per iteration, one short extra round).  Three __syncwarp()s per round
//     order the phases; nothing in the hot loop is an atomic.
//   * HBM latency: DEPTH row quads per lane are in flight in registers, and every warp prefetches its column chunks
//     WP_PF_STAGES iterations ahead into L2 (prefetch.global.L2 -> CCTL.E.PF2, one line per lane) — two warps per
//     scheduler cannot cover a ~1.5 us loaded HBM latency with registers alone.
//   * flush: the CTA adds its warps' tables per id and merges ONE partial per group into the global table
//     (AggFnCall::merge semantics, same as the lean kernel's flush).
//
// Shape (checked by the host, api.cu): NULL-free batch, predicate terms `int32 column <cmp> int32 constant`, a 4-byte
// integer key column (or, with JOIN, a 4-byte foreign key resolved through the JoinProbe), at most two 8-byte value
// columns each feeding exactly one SUM lane (double or int64); COUNT(*) / AVG ride on the row count.  Everything else
// stays on k_agg_group_lean / k_agg_group_direct.  Groups beyond the per-warp capacity (ids >= wp_gcap) take the
// global-table path row by row — correct for any cardinality, and the host switches kernels when it learns the
// cardinality is too high.
//
// Replaces FilterNode::need_copy + AggNode::process_row_batch + AggFnCall::update for one column batch
// (/root/reference/src/exec/filter_node.cpp:726-795, src/exec/agg_node.cpp:507-545, src/expr/agg_fn_call.cpp:496-555).
#pragma once
#include "agg_direct.cuh"

namespace bk {

// warps per CTA: each SM sub-partition has 16K registers, so 8 warps (two per scheduler) may use 248 registers, 12 warps 168,
// 16 warps 128; the table memory (one accumulator set per warp) decides how many fit
constexpr int wp_regs(int warps) { return warps <= 8 ? 248 : (warps <= 12 ? 168 : 128); }
constexpr uint32_t WP_TAG_BITS = 8;          // low bits of a count word: arbitration tag (entry slot * 32 + lane)
constexpr uint32_t WP_TAG_MASK = (1u << WP_TAG_BITS) - 1u;   // rows per (warp, group, launch) < 2^24 (a CTA sees < 2^30 / grid rows)
constexpr uint32_t WP_PENDING = 0xFFFFFFFEu; // id of a key-table entry whose id is being assigned
constexpr uint32_t WP_NOID = 0xFFFFFFF0u;    // "no dense id": the row goes to the global table
constexpr int WP_PF_ITERS = 3;               // L2 prefetch distance in warp iterations (two chunks each) beyond the register stage

__device__ __forceinline__ uint32_t wp_lds32(uint32_t a) { uint32_t v; asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void wp_sts64(uint32_t a, uint64_t v) { asm volatile("st.volatile.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ void wp_lds128(uint32_t a, uint64_t& lo, uint64_t& hi) { asm volatile("ld.volatile.shared.v2.u64 {%0,%1}, [%2];" : "=l"(lo), "=l"(hi) : "r"(a) : "memory"); }
// predicated forms (PTX guard predicates: ptxas keeps them as @P LDS / @P STS instead of branching around each access)
__device__ __forceinline__ uint32_t wp_lds32_if(uint32_t a, bool on) {
    uint32_t v; asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %2, 0;\n @p ld.volatile.shared.u32 %0, [%1];\n}" : "=r"(v) : "r"(a), "r"((uint32_t)on) : "memory"); return v;
}
__device__ __forceinline__ void wp_sts32_if(uint32_t a, uint32_t v, bool on) {
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %2, 0;\n @p st.volatile.shared.u32 [%0], %1;\n}" ::"r"(a), "r"(v), "r"((uint32_t)on) : "memory");
}
__device__ __forceinline__ uint64_t wp_lds64_if(uint32_t a, bool on) {
    uint64_t v; asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %2, 0;\n @p ld.volatile.shared.u64 %0, [%1];\n}" : "=l"(v) : "r"(a), "r"((uint32_t)on) : "memory"); return v;
}
__device__ __forceinline__ void wp_sts64_if(uint32_t a, uint64_t v, bool on) {
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %2, 0;\n @p st.volatile.shared.u64 [%0], %1;\n}" ::"r"(a), "l"(v), "r"((uint32_t)on) : "memory");
}
__device__ __forceinline__ void wp_lds128_if(uint32_t a, uint64_t& lo, uint64_t& hi, bool on) {
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %3, 0;\n @p ld.volatile.shared.v2.u64 {%0,%1}, [%2];\n}" : "=l"(lo), "=l"(hi) : "r"(a), "r"((uint32_t)on) : "memory");
}
__device__ __forceinline__ void wp_sts128_if(uint32_t a, uint64_t lo, uint64_t hi, bool on) {
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %3, 0;\n @p st.volatile.shared.v2.u64 [%0], {%1,%2};\n}" ::"r"(a), "l"(lo), "l"(hi), "r"((uint32_t)on) : "memory");
}
__device__ __forceinline__ void wp_prefetch_l2_if(const void* p, bool on) {
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %1, 0;\n @p prefetch.global.L2 [%0];\n}" ::"l"(p), "r"((uint32_t)on));
}

__device__ __forceinline__ size_t wp_warp_bytes_dev(int na, uint32_t gcap) { return ((size_t)gcap * (8u * (uint32_t)na + 4u) + 15) & ~(size_t)15; }

// rare path: claim an EMPTY key-table word for `key`.  Returns the new id, or WP_PENDING when another lane / warp took
// the word first (the caller examines the bucket again), or WP_NOID when the table is too full to take more keys.
__device__ __forceinline__ uint32_t wp_insert(uint32_t slot_addr, uint32_t key, uint32_t next_id_addr, uint32_t id_limit) {
    if (wp_lds32(next_id_addr) >= id_limit) return WP_NOID;
    const uint64_t old = atoms_cas64(slot_addr, ~0ull, (uint64_t)key | ((uint64_t)WP_PENDING << 32));
    if (old != ~0ull) return WP_PENDING;
    const uint32_t id = atoms_add32(next_id_addr, 1u);
    wp_sts64(slot_addr, (uint64_t)key | ((uint64_t)id << 32));
    return id;
}

// rare path: a row whose group has no dense id in this CTA updates the global table directly (inlined once per stage — a
// call inside the hot loop makes ptxas park the in-flight column registers in local memory around it)
template <int NA>
__device__ __forceinline__ void wp_global_row(const AggArgs& a, uint32_t key, uint64_t v0, uint64_t v1) {
    const AggPlan& ap = a.plan;
    const GroupTable& gt = a.gt;
    const uint32_t gcap = gt.cap_mask + 1;
    uint64_t gk[MAX_KEYW];
    gk[0] = (uint64_t)key;
    for (int w = 1; w < ap.n_keyw; w++) gk[w] = 0ull;
    const int slot = table_upsert<false, 0>(gt.state, gt.keys, gt.cap_mask, gk, ap.n_keyw, ap.n_keyw == 1 ? hash_key1(gk[0]) : hash_key(gk, ap.n_keyw), (int)gcap, gt.n_groups);
    if (slot < 0) { atomicExch(gt.overflow, 1u); return; }
    atomicAdd((unsigned long long*)(gt.lanes + slot), 1ull);
#pragma unroll
    for (int s = 0; s < NA; s++) {
        const uint64_t v = s == 0 ? v0 : v1;
        // the column's non-NULL counter (AVG's count): the flush fills it from the row count, a row on this path adds its own
        if (a.vops[s].cnt_glob) atomicAdd((unsigned long long*)(gt.lanes + (size_t)a.vops[s].cnt_glob * gcap + slot), 1ull);
        uint64_t* p = gt.lanes + (size_t)a.vops[s].glob_lane[0] * gcap + slot;
        if (a.vops[s].op[0] == LN_ADD_F64) atomicAdd((double*)p, bits_f64(v)); else atomicAdd((unsigned long long*)p, (unsigned long long)v);
    }
}


// ------------------------------------------------------------------------------------------------------------------
// The two hot blocks of the loop (first key-table probe, arbitration round) are written in PTX for WP_E = 8 entry slots per
// lane — generated by csrc/gen_wp_ptx.py.  nvcc materialises every `bool` that guards an inline-asm access as SEL + ISETP,
// which more than doubled the instruction count of the C++ statement of the same steps.
// Flags travel between the blocks as bit masks (bit j = entry slot j of this lane).
// ------------------------------------------------------------------------------------------------------------------
#include "agg_wp_ptx.inc"

// element j of a register array by a run-time index without touching local memory (select chain)
template <class V>
__device__ __forceinline__ V wp_sel8(const V (&x)[8], int j) {
    const V lo = j & 2 ? (j & 1 ? x[3] : x[2]) : (j & 1 ? x[1] : x[0]);
    const V hi = j & 2 ? (j & 1 ? x[7] : x[6]) : (j & 1 ? x[5] : x[4]);
    return j & 4 ? hi : lo;
}

// `int32 column <cmp> int32 constant` as ((x ^ m) <u t) != flip: LT / GE compare in the biased domain (m = 2^31), EQ / NE test
// (x ^ c) <u 1, LE / GT use c + 1 (c = INT32_MAX: constant result).  One LOP3 + one ISETP per row whatever the operator.
struct WpTerm { uint32_t m, t; bool flip; };
__device__ __forceinline__ WpTerm wp_term(int cmp, int32_t c) {
    WpTerm w;
    switch (cmp) {
        case BK_FT_EQ: w.m = (uint32_t)c; w.t = 1u; w.flip = false; break;
        case BK_FT_NE: w.m = (uint32_t)c; w.t = 1u; w.flip = true; break;
        case BK_FT_LT: w.m = 0x80000000u; w.t = (uint32_t)c ^ 0x80000000u; w.flip = false; break;
        case BK_FT_GE: w.m = 0x80000000u; w.t = (uint32_t)c ^ 0x80000000u; w.flip = true; break;
        case BK_FT_LE: w.m = 0x80000000u; w.t = c == INT32_MAX ? 0u : ((uint32_t)(c + 1) ^ 0x80000000u); w.flip = c == INT32_MAX; break;
        default /*GT*/: w.m = 0x80000000u; w.t = c == INT32_MAX ? 0u : ((uint32_t)(c + 1) ^ 0x80000000u); w.flip = c != INT32_MAX; break;
    }
    return w;
}

template <int NP, int NA, bool JOIN, bool F64, bool DENSE, int WARPS>
__global__ void __maxnreg__(wp_regs(WARPS)) k_agg_group_wp(const __grid_constant__ AggArgs a) {
    static_assert(NA <= 2, "warp-private kernel: at most two value columns");
    constexpr int S1 = NA > 1 ? 1 : 0;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const AggPlan& ap = a.plan;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t G = (uint32_t)a.wp_gcap;
    const uint32_t kt_cap = DENSE ? 0u : (1u << a.wp_kt_log2);            // words; buckets of two
    const uint32_t bk_mask = (kt_cap >> 1) - 1u;
    const int hash_shift = 33 - a.wp_kt_log2;
    const uint32_t id_limit = kt_cap - (kt_cap >> 2);                      // the key table takes keys up to 75 % load
    uint64_t* kt = (uint64_t*)smem_raw;
    uint32_t* next_id = (uint32_t*)(kt + kt_cap);
    const size_t wbytes = wp_warp_bytes_dev(NA, G);
    unsigned char* acc0 = (unsigned char*)(next_id + 4);
    // ---- init: key table EMPTY, every warp zeroes its own accumulators (the identity of ADD and of the row count) ----
    if constexpr (!DENSE) { for (uint32_t i = threadIdx.x; i < kt_cap; i += blockDim.x) kt[i] = ~0ull; }
    if (threadIdx.x == 0) *next_id = 0;
    {
        uint32_t* w = (uint32_t*)(acc0 + wbytes * warp);
        for (uint32_t i = lane; i < wbytes / 4; i += 32) w[i] = 0u;
    }
    __syncthreads();
    const uint32_t kt_addr = smem_addr(kt), nid_addr = smem_addr(next_id);
    const uint32_t sums_addr = smem_addr(acc0 + wbytes * warp);
    const uint32_t cnt_addr = sums_addr + G * 8u * NA;
    const uint32_t dense_sub = (uint32_t)a.wp_dense_sub;                  // DENSE: id = key - dense_sub (mod 2^32)

    const uint32_t kmask = ap.key_bits[0] >= 32 ? 0xFFFFFFFFu : ((1u << ap.key_bits[0]) - 1u);
    WpTerm term[NP > 0 ? NP : 1];
    const uint8_t* tptr[NP > 0 ? NP : 1];
#pragma unroll
    for (int t = 0; t < NP; t++) { term[t] = wp_term(a.direct.term[t].cmp, (int32_t)(int64_t)a.direct.term[t].cbits); tptr[t] = (const uint8_t*)a.cols[t].values; }
    const uint8_t* kptr = (const uint8_t*)a.cols[NP].values;
    const uint8_t* vptr[NA > 0 ? NA : 1]; bool acc_f64[NA > 0 ? NA : 1];
#pragma unroll
    for (int s = 0; s < NA; s++) { vptr[s] = (const uint8_t*)a.cols[NP + 1 + s].values; acc_f64[s] = F64 || a.vops[s].op[0] == LN_ADD_F64; }
    const uint32_t tag0 = (1u << WP_TAG_BITS) + (uint32_t)lane;   // entry slot j writes (count + 1) << 8 | (j * 32 + lane)

    // this lane's L2 prefetch duty: one 128-byte line of one column chunk per chunk
    // (a 4-byte column chunk of 32 quads is 512 B = 4 lines, an 8-byte column chunk 1 KB = 8 lines)
    const uint8_t* pf_base = nullptr; uint32_t pf_mul = 0;
    {
        int l = lane;
#pragma unroll
        for (int c = 0; c < NP + 1 + NA; c++) {
            const int lines = c <= NP ? 4 : 8;
            if (l >= 0 && l < lines) { pf_base = (c < NP ? tptr[c < NP ? c : 0] : (c == NP ? kptr : vptr[c > NP ? c - NP - 1 : 0])) + l * 128; pf_mul = c <= NP ? 16u : 32u; }
            l -= lines;
        }
    }

    uint32_t passed = 0;
    const uint32_t nquads = (uint32_t)(a.nrows >> 2);                        // (a launch covers < 2^30 rows)
    const uint32_t T = blockDim.x;
    const uint32_t stride = gridDim.x * T;                                  // quads between two chunks of a warp
    const uint32_t qw = blockIdx.x * T + warp * 32;                         // first quad of this warp's first chunk
    const uint32_t chunks = qw < nquads ? (nquads - qw + stride - 1) / stride : 0u;   // (warp-uniform)
    const uint32_t iters = (chunks + 1) >> 1;                               // two chunks (row quads A and B of a lane) per iteration
    const uint32_t qlast = nquads ? nquads - 1 : 0;
    // one register stage: the raw columns of quad A = qw + 2 * it * stride + lane and quad B = A + stride.  The stage is copied
    // out and refilled for the next iteration before its rows are aggregated, so the loads fly for a whole iteration.  Loads are
    // never guarded: a quad index past the end is clamped to the last quad (the rows are masked out where they are used).
    uint32_t pr[2][NP > 0 ? NP : 1][4]; uint32_t kr[2][4]; uint64_t vr[2][NA > 0 ? NA : 1][4];
    auto issue_loads = [&](int h, uint32_t q) {
        q = q < qlast ? q : qlast;
#pragma unroll
        for (int t = 0; t < NP; t++) { const U32x4 r = ldg128_u32(tptr[t] + (size_t)q * 16);
#pragma unroll
            for (int j = 0; j < 4; j++) pr[h][t][j] = r.v[j]; }
        { const U32x4 r = ldg128_u32(kptr + (size_t)q * 16);
#pragma unroll
            for (int j = 0; j < 4; j++) kr[h][j] = r.v[j]; }
#pragma unroll
        for (int s = 0; s < NA; s++) { const U64x4 r = ldg256_u64(vptr[s] + (size_t)q * 32);
#pragma unroll
            for (int j = 0; j < 4; j++) vr[h][s][j] = r.v[j]; }
    };
    auto prefetch_chunk = [&](uint32_t c) {   // chunk c of this warp: quads [qw + c * stride, + 32)
        const uint32_t qp = qw + c * stride;
        wp_prefetch_l2_if(pf_base + (size_t)qp * pf_mul, pf_base != nullptr && c < chunks && qp + 32 <= nquads);
    };
    if (nquads) {
        issue_loads(0, qw + lane); issue_loads(1, qw + stride + lane);
#pragma unroll
        for (int c = 2; c < 2 + 2 * WP_PF_ITERS; c++) prefetch_chunk(c);
    }

#pragma unroll 1
    for (uint32_t it = 0; it < iters; it++) {
        const uint32_t qa = qw + 2 * it * stride + lane, qb = qa + stride;
        // ---- filter (FilterNode::need_copy): bit j of `act` = row j of quad A, bit 4 + j = row j of quad B ----
        uint32_t act = (qa < nquads ? 0x0Fu : 0u) | ((2 * it + 1 < chunks && qb < nquads) ? 0xF0u : 0u);
#pragma unroll
        for (int t = 0; t < NP; t++) {
            uint32_t m = 0;
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
                for (int j = 0; j < 4; j++) m |= ((((pr[h][t][j] ^ term[t].m) < term[t].t) != term[t].flip) ? 1u : 0u) << (4 * h + j);
            act &= m;
        }
        uint32_t key[8]; uint64_t v[NA > 0 ? NA : 1][8];
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int j = 0; j < 4; j++) {
                key[4 * h + j] = kr[h][j];
#pragma unroll
                for (int s = 0; s < NA; s++) v[s][4 * h + j] = vr[h][s][j];
            }
        // ---- the stage is copied out: refill it, and start two chunks WP_PF_ITERS iterations further on their way into L2 ----
        if (it + 1 < iters) { issue_loads(0, qa + 2 * stride); issue_loads(1, qb + 2 * stride); }
        prefetch_chunk(2 * (it + 1 + WP_PF_ITERS)); prefetch_chunk(2 * (it + 1 + WP_PF_ITERS) + 1);
        if (JOIN) {   // K4 fused: foreign key -> dimension attribute (one L2-resident read per surviving row), inner join
            const JoinProbe& jp = a.jp;
            uint32_t g[8];
            if (jp.mode == 1) {
                uint64_t off[8];
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const uint64_t img = jp.key_signed ? (uint64_t)(int64_t)(int32_t)key[j] : (uint64_t)key[j];
                    off[j] = (img ^ jp.bias) - jp.dense_min;
                    if (off[j] >= jp.dense_size) act &= ~(1u << j);
                }
#pragma unroll
                for (int j = 0; j < 8; j++) g[j] = ((act >> j) & 1u) ? __ldg(jp.attr + off[j]) : 0u;
                if (jp.present) {
                    uint32_t pr8[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) pr8[j] = ((act >> j) & 1u) ? __ldg(jp.present + off[j]) : 0xFFFFFFFFu;
#pragma unroll
                    for (int j = 0; j < 8; j++) if (pr8[j] == 0xFFFFFFFFu) act &= ~(1u << j);
                }
            } else {
                uint32_t slot[8]; uint64_t e[8];
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    slot[j] = (key[j] * 0x9E3779B1u) & jp.packed_mask;
                    e[j] = ((act >> j) & 1u) ? __ldg((const unsigned long long*)(jp.packed + slot[j])) : ~0ull;
                }
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    g[j] = 0; bool hit = false;
                    while (e[j] != ~0ull) {
                        if ((uint32_t)(e[j] >> 32) == key[j]) { g[j] = (uint32_t)e[j]; hit = true; break; }
                        slot[j] = (slot[j] + 1) & jp.packed_mask;
                        e[j] = __ldg((const unsigned long long*)(jp.packed + slot[j]));
                    }
                    if (!hit) act &= ~(1u << j);
                }
            }
#pragma unroll
            for (int j = 0; j < 8; j++) key[j] = g[j];
        }
#pragma unroll
        for (int j = 0; j < 8; j++) key[j] &= kmask;
        passed += __popc(act);

        // ---- key -> dense id ----
        uint32_t id[8];
        if (DENSE) {
#pragma unroll
            for (int j = 0; j < 8; j++) id[j] = key[j] - dense_sub;
        } else {
            // the first probe is branch-free (wp_probe8); only displaced keys, first sightings and ids in flight enter the loop:
            // every lane works on its lowest unresolved entry, one bucket look per trip (no lane ever spins on another lane)
            uint32_t need = wp_probe8(act, key, kt_addr, (uint32_t)hash_shift, id);
            if (__any_sync(0xFFFFFFFFu, need != 0)) {
                uint32_t cur = 0xFFu, kc = 0, bkc = 0;
                do {
                    if (need) {
                        const uint32_t j = (uint32_t)__ffs((int)need) - 1u;
                        if (j != cur) { cur = j; kc = wp_sel8(key, (int)j); bkc = (kc * 0x9E3779B1u) >> hash_shift; }
                        const uint32_t baddr = kt_addr + bkc * 16u;
                        uint64_t e0, e1;
                        wp_lds128(baddr, e0, e1);
                        uint32_t r = WP_PENDING;                                   // PENDING = look at this bucket again
                        if (e0 == ~0ull) r = wp_insert(baddr, kc, nid_addr, id_limit);          // free word: first row of this key in the CTA
                        else if ((uint32_t)e0 == kc) r = (uint32_t)(e0 >> 32);                    // (PENDING: its owner publishes the id)
                        else if (e1 == ~0ull) r = wp_insert(baddr + 8u, kc, nid_addr, id_limit);
                        else if ((uint32_t)e1 == kc) r = (uint32_t)(e1 >> 32);
                        else bkc = (bkc + 1) & bk_mask;
                        if (r != WP_PENDING) {                                     // (WP_NOID: global path)
#pragma unroll
                            for (int i = 0; i < 8; i++) id[i] = (uint32_t)i == j ? r : id[i];
                            need &= need - 1u;
                        }
                    }
                } while (__any_sync(0xFFFFFFFFu, need != 0));
            }
        }
        // ---- groups beyond the per-warp capacity: straight to the global table (rare) ----
        uint32_t pend = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) pend |= (id[j] < G ? 1u : 0u) << j;
        pend &= act;
        if (__any_sync(0xFFFFFFFFu, pend != act)) {
            uint32_t ovf = act & ~pend;
            while (ovf) {
                const int j = __ffs((int)ovf) - 1;
                ovf &= ovf - 1u;
                wp_global_row<NA>(a, wp_sel8(key, j), NA > 0 ? wp_sel8(v[0], j) : 0ull, NA > 1 ? wp_sel8(v[S1], j) : 0ull);
            }
        }
        // ---- accumulate: rounds of {read cnt | write cnt + 1 with my tag | read back | winners add their values} ----
        uint64_t ad[8];   // count word address | sums address << 32
#pragma unroll
        for (int j = 0; j < 8; j++) ad[j] = (uint64_t)(cnt_addr + id[j] * 4u) | ((uint64_t)(sums_addr + id[j] * (8u * NA)) << 32);
        if (F64 && NA == 2) {
            do pend = wp_round8_f64x2(pend, ad, tag0, v[0], v[S1]); while (__any_sync(0xFFFFFFFFu, pend != 0));
        } else if (F64 && NA == 1) {
            do pend = wp_round8_f64x1(pend, ad, tag0, v[0]); while (__any_sync(0xFFFFFFFFu, pend != 0));
        } else {
            do {   // (integer sums / COUNT(*) only: the C++ statement of the same round)
                uint32_t mine[8];
#pragma unroll
                for (int j = 0; j < 8; j++) mine[j] = wp_lds32_if((uint32_t)ad[j], (pend >> j) & 1u);
                __syncwarp();
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    mine[j] = (mine[j] & ~WP_TAG_MASK) + tag0 + 32u * j;
                    wp_sts32_if((uint32_t)ad[j], mine[j], (pend >> j) & 1u);
                }
                __syncwarp();
                uint32_t win = 0;
#pragma unroll
                for (int j = 0; j < 8; j++) win |= (wp_lds32_if((uint32_t)ad[j], (pend >> j) & 1u) == mine[j] ? 1u : 0u) << j;
                win &= pend;
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const uint32_t sa = (uint32_t)(ad[j] >> 32);
                    if (NA == 2) {
                        uint64_t s0, s1;
                        wp_lds128_if(sa, s0, s1, (win >> j) & 1u);
                        const uint64_t n0 = acc_f64[0] ? f64_bits(bits_f64(s0) + bits_f64(v[0][j])) : s0 + v[0][j];
                        const uint64_t n1 = acc_f64[S1] ? f64_bits(bits_f64(s1) + bits_f64(v[S1][j])) : s1 + v[S1][j];
                        wp_sts128_if(sa, n0, n1, (win >> j) & 1u);
                    } else if (NA == 1) {
                        const uint64_t s0 = wp_lds64_if(sa, (win >> j) & 1u);
                        wp_sts64_if(sa, acc_f64[0] ? f64_bits(bits_f64(s0) + bits_f64(v[0][j])) : s0 + v[0][j], (win >> j) & 1u);
                    }
                }
                pend &= ~win;
                __syncwarp();
            } while (__any_sync(0xFFFFFFFFu, pend != 0));
        }
    }

    // ---- flush: one partial per group and CTA into the global table (AggFnCall::merge) ----
    __syncthreads();
    {
        const int nwarps = blockDim.x >> 5;
        const GroupTable& gt = a.gt;
        int glane[NA > 0 ? NA : 1];
#pragma unroll
        for (int s = 0; s < NA; s++) glane[s] = a.vops[s].glob_lane[0];
        const uint32_t n_scan = DENSE ? G : kt_cap;
        for (uint32_t i = threadIdx.x; i < n_scan; i += blockDim.x) {
            uint32_t gid, gkey;
            if (DENSE) { gid = i; gkey = i + dense_sub; }
            else {
                const uint64_t e = kt[i];
                if (e == ~0ull) continue;
                gid = (uint32_t)(e >> 32); gkey = (uint32_t)e;
                if (gid >= G) continue;
            }
            uint64_t rows = 0; uint64_t sum[NA > 0 ? NA : 1];
#pragma unroll
            for (int s = 0; s < NA; s++) sum[s] = 0ull;   // +0.0 == 0 bits: identity for both ADD flavours
            for (int w = 0; w < nwarps; w++) {
                const unsigned char* wb = acc0 + wbytes * w;
                const uint32_t c = ((const uint32_t*)(wb + (size_t)G * 8u * NA))[gid] >> WP_TAG_BITS;
                if (!c) continue;
                rows += c;
#pragma unroll
                for (int s = 0; s < NA; s++) {
                    const uint64_t x = ((const uint64_t*)wb)[(size_t)gid * NA + s];
                    sum[s] = acc_f64[s] ? f64_bits(bits_f64(sum[s]) + bits_f64(x)) : sum[s] + x;
                }
            }
            if (!rows) continue;
            uint64_t key[MAX_KEYW];
            key[0] = (uint64_t)gkey;
            for (int w = 1; w < ap.n_keyw; w++) key[w] = 0ull;
            merge_group(ap, gt, key, [&](int l, uint64_t& val) {
                if (l == 0 || ((a.alias_mask >> l) & 1u)) { val = rows; return true; }
#pragma unroll
                for (int s = 0; s < NA; s++) if (l == glane[s]) { val = sum[s]; return true; }
                return false;
            });
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (a.nrows & 3)) passed += direct_tail_row<NP, NA, JOIN>(a, (a.nrows & ~(int64_t)3) + threadIdx.x);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) passed += __shfl_xor_sync(0xFFFFFFFFu, passed, d);
    if (lane == 0 && passed) atomicAdd((unsigned long long*)a.rows_passed, (unsigned long long)passed);
}

template <int NP, int NA, bool JOIN, bool F64, bool DENSE, int WARPS>
static inline cudaError_t launch_wp_k(const AggArgs& a, int sm_count, cudaStream_t s, cudaEvent_t start) {
    const size_t smem = wp_smem_bytes(NA, (uint32_t)a.wp_gcap, a.wp_dense ? -1 : a.wp_kt_log2, WARPS);
    const int64_t want = ((a.nrows + 3) / 4 + WARPS * 32 - 1) / (WARPS * 32);
    const int grid = (int)(want < sm_count ? want : sm_count);   // persistent: one CTA per SM
    cudaError_t e = cudaFuncSetAttribute(k_agg_group_wp<NP, NA, JOIN, F64, DENSE, WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (start) cudaEventRecord(start, s);
    k_agg_group_wp<NP, NA, JOIN, F64, DENSE, WARPS><<<grid, WARPS * 32, smem, s>>>(a);
    return cudaGetLastError();
}
template <int NP, int NA, bool JOIN, bool F64, bool DENSE>
static inline cudaError_t launch_wp_w(const AggArgs& a, int sm_count, cudaStream_t s, cudaEvent_t start) {
    if constexpr (NA <= 1) {   // (two value columns: 20 bytes per group and warp — more than eight tables never fit a useful capacity)
        if (a.wp_warps == 16) return launch_wp_k<NP, NA, JOIN, F64, DENSE, 16>(a, sm_count, s, start);
        if (a.wp_warps == 12) return launch_wp_k<NP, NA, JOIN, F64, DENSE, 12>(a, sm_count, s, start);
    }
    return launch_wp_k<NP, NA, JOIN, F64, DENSE, 8>(a, sm_count, s, start);
}
template <int NP, int NA, bool JOIN, bool F64>
static inline cudaError_t launch_wp_d(const AggArgs& a, int sm_count, cudaStream_t s, cudaEvent_t start) {
    return a.wp_dense ? launch_wp_w<NP, NA, JOIN, F64, true>(a, sm_count, s, start) : launch_wp_w<NP, NA, JOIN, F64, false>(a, sm_count, s, start);
}

template <int NP, int NA>
static inline cudaError_t launch_wp(const AggArgs& a, int sm_count, cudaStream_t s, cudaEvent_t start) {
    if constexpr (NA <= 2) {
        bool all_f64 = true;   // every value column feeds a double sum: the adds are compiled in (no per-entry type select)
        for (int v = 0; v < NA; v++) all_f64 = all_f64 && a.vops[v].op[0] == LN_ADD_F64;
        if (a.jp.mode) return all_f64 ? launch_wp_d<NP, NA, true, true>(a, sm_count, s, start) : launch_wp_d<NP, NA, true, false>(a, sm_count, s, start);
        return all_f64 ? launch_wp_d<NP, NA, false, true>(a, sm_count, s, start) : launch_wp_d<NP, NA, false, false>(a, sm_count, s, start);
    } else {
        (void)a; (void)sm_count; (void)s; (void)start;
        return cudaErrorInvalidValue;
    }
}

}  // namespace bk

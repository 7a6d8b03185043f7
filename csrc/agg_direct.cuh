// agg_direct.cuh — the specialised filter+aggregate kernels (K1+K2) for the canonical shape:
//   predicate = conjunction of NP terms `column <cmp> constant`, GROUP BY one column (or none),
//   aggregate arguments = NA plain columns.  args.cols[] is ordered [NP predicate][key][NA value]
//   columns by the host, so every slot index below is a compile-time constant.
//
// Structure of one warp iteration (128 rows = 4 consecutive rows per lane):
//   1. LOAD     one 128-bit (4-byte types) or 256-bit (8-byte types) non-allocating load per column,
//               issued one iteration AHEAD (software prefetch: loads fly while atomics run)
//   2. FILTER   predicate in registers -> 4-bit pass mask per lane          (FilterNode::need_copy)
//   3. COMPACT  four warp ballots give every surviving row its position in a per-warp queue in
//               shared memory (key + NA values + null bits)                 [warp-ballot stream compaction]
//   4. CONSUME  all 32 lanes drain the queue: probe the per-CTA hash table, then shared-memory
//               atomics on the group's lanes                                (AggFnCall::update)
// Step 3 removes the selectivity-dependent lane divergence from step 4 and keeps the kernel small
// enough for the instruction cache (the first version unrolled the aggregate step 8x per thread,
// grew to 15k SASS instructions and lost most of its issue slots to instruction fetch).  Everything the loop needs from the plan descriptors is
// resolved into registers before the loop; uncommon shapes (min/max, float/bool/narrow columns,
// NULL keys wider than 32 bits ...) take out-of-line routines so the hot loop stays lean.
#pragma once
#include <map>
#include <mutex>
#include <tuple>
#include "agg_kernels.cuh"
#include "agg_select.h"
#include "fx.h"

namespace bk {

constexpr int ROWS_PER_LANE = 4;
constexpr int QCAP = 32 * ROWS_PER_LANE;  // queue entries per warp
constexpr int LEAN_QCAP = QCAP + 32;      // the lean kernel's ring: one iteration's survivors + the < 32 carried over

// per-column decode flags, computed once per kernel
enum : uint32_t { SF_IS8 = 1u, SF_SIGNED = 2u, SF_SPECIAL = 4u, SF_HASV = 8u };
__device__ __forceinline__ uint32_t slot_flags(const DevCol& c) {
    uint32_t f = 0;
    if (c.stype == ST_I64 || c.stype == ST_U64 || c.stype == ST_F64) f |= SF_IS8;
    if (c.stype == ST_I32) f |= SF_SIGNED;
    if (c.stype == ST_F32 || c.stype == ST_U8 || c.prim == BK_INT8 || c.prim == BK_INT16 || c.prim == BK_UINT8 ||
        c.prim == BK_UINT16 || c.prim == BK_BOOL) f |= SF_SPECIAL;
    if (c.validity) f |= SF_HASV;
    return f;
}

struct RawQuad { uint32_t r[8]; uint32_t nm; };

// four consecutive rows [4q, 4q+4) of one column (full quads only: the <= 3 ragged rows at the end of a
// batch are handled by direct_tail_row)
__device__ __forceinline__ void raw_quad_load(const DevCol& c, uint32_t flags, int64_t q, RawQuad& out) {
    if (flags & SF_IS8) {
        const U32x8 r = ldg256_u32((const uint8_t*)c.values + q * 32);
#pragma unroll
        for (int j = 0; j < 8; j++) out.r[j] = r.v[j];
    } else if (c.stype == ST_U8) {
        out.r[0] = __ldg((const uint32_t*)c.values + q);
    } else {
        asm("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
            : "=r"(out.r[0]), "=r"(out.r[1]), "=r"(out.r[2]), "=r"(out.r[3]) : "l"((const uint8_t*)c.values + q * 16));
    }
    out.nm = 0;
    if (flags & SF_HASV) out.nm = (~((uint32_t)__ldg(c.validity + (q >> 1)) >> ((q & 1) * 4))) & 0xFu;
}
// float / bool / narrow integer columns: rare, decoded through the general switch
__device__ __forceinline__ uint64_t decode_special(uint32_t r, int j, int stype, int prim) {
    uint64_t v;
    switch (stype) {
        case ST_F32: v = f64_bits((double)__uint_as_float(r)); break;
        case ST_U8: v = (r >> (8 * j)) & 0xFFu; break;
        case ST_I32: v = (uint64_t)(int64_t)(int32_t)r; break;
        default: v = r; break;
    }
    return narrow_prim(v, prim);
}
__device__ __forceinline__ void raw_quad_decode(const RawQuad& in, uint32_t flags, const DevCol& c, uint64_t (&v)[4]) {
    if (flags & SF_IS8) {
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = (uint64_t)in.r[2 * j] | ((uint64_t)in.r[2 * j + 1] << 32);
    } else if (!(flags & SF_SPECIAL)) {  // int32 / uint32: branch-free sign or zero extension
        const uint32_t sm = (flags & SF_SIGNED) ? 0xFFFFFFFFu : 0u;
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = (uint64_t)in.r[j] | ((uint64_t)((uint32_t)((int32_t)in.r[j] >> 31) & sm) << 32);
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = decode_special(c.stype == ST_U8 ? in.r[0] : in.r[j], j, c.stype, c.prim);
    }
}

// `column <cmp> constant` over four rows -> 4-bit mask; one switch per quad, tight loops inside.
// IEEE semantics for DOUBLE (NaN fails every ordered compare, != holds): operators.cpp:84-100.
#define BK_CMP4(T, EXPR)                                                                    \
    {                                                                                       \
        _Pragma("unroll") for (int j = 0; j < 4; j++) { const T x = (T)xs[j]; m |= ((EXPR) ? 1u : 0u) << j; } \
    }                                                                                       \
    break;
__device__ __forceinline__ uint32_t term_mask(const DirectTerm& t, const uint64_t (&v)[4]) {
    uint32_t m = 0;
    if (t.vclass == VC_F64) {
        double xs[4];
#pragma unroll
        for (int j = 0; j < 4; j++) xs[j] = bits_f64(v[j]);
        const double y = bits_f64(t.cbits);
        switch (t.cmp) {
            case BK_FT_EQ: BK_CMP4(double, x == y) case BK_FT_NE: BK_CMP4(double, x != y)
            case BK_FT_LT: BK_CMP4(double, x < y) case BK_FT_LE: BK_CMP4(double, x <= y)
            case BK_FT_GT: BK_CMP4(double, x > y) default: BK_CMP4(double, x >= y)
        }
    } else if (t.vclass == VC_U64) {
        const uint64_t* xs = v; const uint64_t y = t.cbits;
        switch (t.cmp) {
            case BK_FT_EQ: BK_CMP4(uint64_t, x == y) case BK_FT_NE: BK_CMP4(uint64_t, x != y)
            case BK_FT_LT: BK_CMP4(uint64_t, x < y) case BK_FT_LE: BK_CMP4(uint64_t, x <= y)
            case BK_FT_GT: BK_CMP4(uint64_t, x > y) default: BK_CMP4(uint64_t, x >= y)
        }
    } else {
        const uint64_t* xs = v; const int64_t y = (int64_t)t.cbits;
        switch (t.cmp) {
            case BK_FT_EQ: BK_CMP4(int64_t, x == y) case BK_FT_NE: BK_CMP4(int64_t, x != y)
            case BK_FT_LT: BK_CMP4(int64_t, x < y) case BK_FT_LE: BK_CMP4(int64_t, x <= y)
            case BK_FT_GT: BK_CMP4(int64_t, x > y) default: BK_CMP4(int64_t, x >= y)
        }
    }
    return m;
}
#undef BK_CMP4

// read-modify-write of one 8-byte lane in shared memory with a CAS loop (min / max of any class)
static __device__ __noinline__ void smem_rmw(int op, uint64_t* p, uint64_t v) {
    unsigned long long* q = (unsigned long long*)p;
    unsigned long long cur = *(volatile unsigned long long*)q;
    for (;;) {
        const unsigned long long nw = lane_combine(op, cur, v);
        if (nw == cur) break;
        const unsigned long long prev = atomicCAS(q, cur, nw);
        if (prev == cur) break;
        cur = prev;
    }
}
// double add: LDS + DADD + ATOMS.CAS loop (sm_90a has no native 64-bit floating add in shared memory)
__device__ __forceinline__ void smem_add_f64(uint64_t* p, double v) {
    unsigned long long* q = (unsigned long long*)p;
    unsigned long long cur = *(volatile unsigned long long*)q;
    for (;;) {
        const unsigned long long nw = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)cur) + v);
        const unsigned long long prev = atomicCAS(q, cur, nw);
        if (prev == cur) break;
        cur = prev;
    }
}
__device__ __forceinline__ void smem_lane_update(int op, uint64_t* p, uint64_t v) {
    if (op == LN_ADD_F64) smem_add_f64(p, bits_f64(v));
    else if (op == LN_ADD_I64) smem_add_u64(p, v);
    else smem_rmw(op, p, v);
}
// register accumulation of four rows for the less common lane operations (min / max), out of line
static __device__ __noinline__ uint64_t combine4_generic(int op, uint64_t acc, const uint64_t* v, uint32_t ok, int arg_class, int lane_class) {
    for (int j = 0; j < 4; j++)
        if ((ok >> j) & 1u) acc = lane_combine(op, acc, to_lane_class(v[j], arg_class, lane_class));
    return acc;
}

// a row whose group does not fit the shared table (or when no shared table is in use): update the
// global table directly.  Kept out of line: it is the rare path and must not bloat the hot loop.
template <int NA>
static __device__ __noinline__ void global_update_row(const AggArgs& a, const uint64_t* key, const uint64_t* vals, uint32_t nullbits) {
    const AggPlan& ap = a.plan;
    const GroupTable& gt = a.gt;
    const uint32_t gcap = gt.cap_mask + 1;
    int slot = 0;
    if (ap.n_keyw > 0) {
        slot = table_upsert<false, 0>(gt.state, gt.keys, gt.cap_mask, key, ap.n_keyw,
                                      ap.n_keyw == 1 ? hash_key1(key[0]) : hash_key(key, ap.n_keyw), (int)gcap, gt.n_groups);
        if (slot < 0) { atomicExch(gt.overflow, 1u); return; }
    }
    atomicAdd((unsigned long long*)(gt.lanes + slot), 1ull);
#pragma unroll
    for (int s = 0; s < NA; s++) {
        if ((nullbits >> s) & 1u) continue;
        const ValOps vo = a.vops[s];
        if (vo.cnt_glob) atomicAdd((unsigned long long*)(gt.lanes + (size_t)vo.cnt_glob * gcap + slot), 1ull);
        for (int k = 0; k < vo.n_ops; k++)
            lane_atomic<false>(vo.op[k], gt.lanes + (size_t)vo.glob_lane[k] * gcap + slot, to_lane_class(vals[s], vo.arg_class, vo.lane_class[k]));
    }
}

// uncommon value-column shapes (min / max, several aggregates over one column, int -> double
// conversion): one out-of-line routine per queue entry
template <int NA>
static __device__ __noinline__ void smem_update_row_generic(const AggArgs& a, uint64_t* lanes, uint32_t cap, int slot, const uint64_t* vals, uint32_t nb) {
#pragma unroll
    for (int s = 0; s < NA; s++) {
        if ((nb >> s) & 1u) continue;
        const ValOps vo = a.vops[s];
        if (vo.cnt_smem != 0xFF) atomicAdd((uint32_t*)(lanes + (size_t)vo.cnt_smem * cap + slot), 1u);
        for (int k = 0; k < vo.n_ops; k++)
            smem_lane_update(vo.op[k], lanes + (size_t)vo.smem_lane[k] * cap + slot, to_lane_class(vals[s], vo.arg_class, vo.lane_class[k]));
    }
}

// one of the <= 3 ragged rows at the end of a batch: element loads, straight to the global table
// one foreign key -> dimension attribute (JoinProbe); false = no partner
static __device__ __noinline__ bool join_probe_one(const JoinProbe& jp, uint32_t k, uint32_t& attr) {
    if (jp.mode == 1) {
        const uint64_t img = jp.key_signed ? (uint64_t)(int64_t)(int32_t)k : (uint64_t)k;
        const uint64_t off = (img ^ jp.bias) - jp.dense_min;
        if (off >= jp.dense_size || (jp.present && __ldg(jp.present + off) == 0xFFFFFFFFu)) return false;
        attr = __ldg(jp.attr + off);
        return true;
    }
    uint32_t slot = (k * 0x9E3779B1u) & jp.packed_mask;
    for (;;) {
        const uint64_t e = __ldg((const unsigned long long*)(jp.packed + slot));
        if (e == ~0ull) return false;
        if ((uint32_t)(e >> 32) == k) { attr = (uint32_t)e; return true; }
        slot = (slot + 1) & jp.packed_mask;
    }
}

template <int NP, int NA, bool JOIN = false>
static __device__ __noinline__ uint32_t direct_tail_row(const AggArgs& a, int64_t row) {
    const AggPlan& ap = a.plan;
    for (int t = 0; t < NP; t++) {
        if (elem_is_null(a.cols[t], row)) return 0;
        if (!cmp_vals(a.direct.term[t].cmp, a.direct.term[t].vclass, load_elem(a.cols[t], row), a.direct.term[t].cbits)) return 0;
    }
    uint64_t key[2] = {0, 0};
    int vbase = NP;
    if (ap.n_keyw > 0) {
        const uint64_t kmask = ap.key_bits[0] >= 64 ? ~0ull : ((1ull << ap.key_bits[0]) - 1ull);
        if (JOIN) {   // (lean shape: no NULLs in the batch)
            uint32_t attr = 0;
            if (!join_probe_one(a.jp, (uint32_t)load_elem(a.cols[NP], row), attr)) return 0;
            key[0] = (uint64_t)attr & kmask;
        } else if (elem_is_null(a.cols[NP], row)) key[ap.key_null_word[0] == 1 ? 1 : 0] |= 1ull << ap.key_null_shift[0];
        else key[0] = load_elem(a.cols[NP], row) & kmask;
        vbase = NP + 1;
    }
    uint64_t vals[NA > 0 ? NA : 1]; uint32_t nb = 0;
    for (int s = 0; s < NA; s++) { vals[s] = load_elem(a.cols[vbase + s], row); if (elem_is_null(a.cols[vbase + s], row)) nb |= 1u << s; }
    global_update_row<NA>(a, key, vals, nb);
    return 1;
}

// ------------------------------------------------------------------------------------------
// shared-memory access with 32-bit shared-space addresses: generic pointers cost 64-bit address
// arithmetic plus a generic->shared conversion per access in the hot loop
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint64_t lds64(uint32_t a) { uint64_t v; asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds8(uint32_t a) { uint32_t v; asm volatile("ld.volatile.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts64(uint32_t a, uint64_t v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void reds_inc32(uint32_t a) { asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(a) : "memory"); }
__device__ __forceinline__ uint32_t atoms_add32(uint32_t a, uint32_t v) { uint32_t o; asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(o) : "r"(a), "r"(v) : "memory"); return o; }
__device__ __forceinline__ void lds128(uint32_t a, uint64_t& lo, uint64_t& hi) { asm volatile("ld.volatile.shared.v2.u64 {%0,%1}, [%2];" : "=l"(lo), "=l"(hi) : "r"(a)); }
// 128-bit compare-and-swap in shared memory (ATOMS.CAS.128 on sm_90a): two lanes of a group change together
__device__ __forceinline__ void atoms_cas128(uint32_t a, uint64_t c0, uint64_t c1, uint64_t n0, uint64_t n1, uint64_t& p0, uint64_t& p1) {
    asm volatile("{\n .reg .b128 c, n, p;\n mov.b128 c, {%2, %3};\n mov.b128 n, {%4, %5};\n atom.shared.cas.b128 p, [%6], c, n;\n mov.b128 {%0, %1}, p;\n}"
                 : "=l"(p0), "=l"(p1) : "l"(c0), "l"(c1), "l"(n0), "l"(n1), "r"(a) : "memory");
}
__device__ __forceinline__ uint64_t atoms_cas64(uint32_t a, uint64_t cmp, uint64_t nw) {
    uint64_t o; asm volatile("atom.shared.cas.b64 %0, [%1], %2, %3;" : "=l"(o) : "r"(a), "l"(cmp), "l"(nw) : "memory"); return o;
}
// double add: LDS + DADD + ATOMS.CAS loop (sm_90a has no native 64-bit floating add in shared memory)
__device__ __forceinline__ void smem32_add_f64(uint32_t a, double v) {
    uint64_t cur = lds64(a);
    for (;;) {
        const uint64_t nw = f64_bits(bits_f64(cur) + v);
        const uint64_t prev = atoms_cas64(a, cur, nw);
        if (prev == cur) break;
        cur = prev;
    }
}
// 64-bit integer add from native 32-bit atomics (wraps mod 2^64 like ExprValue::add on INT64)
__device__ __forceinline__ void smem32_add_u64(uint32_t a, uint64_t v) {
    const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
    const uint32_t old = atoms_add32(a, lo);
    const uint32_t carry = (old + lo) < old ? 1u : 0u;
    if (hi + carry) atoms_add32(a + 4, hi + carry);
}
// MIN / MAX in shared memory: compare first, swap only when this value improves the extreme (64-bit min/max atomics are CAS
// loops on sm_90a anyway: ATOMS.CAST.SPIN.64); lane_combine carries the reference's compare semantics (NaN never wins)
__device__ __forceinline__ void smem32_minmax(uint32_t a, int op, uint64_t v) {
    uint64_t cur = lds64(a);
    for (;;) {
        const uint64_t nw = lane_combine(op, cur, v);
        if (nw == cur) break;
        const uint64_t prev = atoms_cas64(a, cur, nw);
        if (prev == cur) break;
        cur = prev;
    }
}
// probe of a sentinel-mode shared table (one-word keys: EMPTY_KEY = free slot): a hit costs one
// LDS.64 and one compare.  Returns the slot's byte offset * 1 (slot index) or -1 after 16 probes.
__device__ __forceinline__ int smem32_upsert1(uint32_t keys_addr, uint32_t cap_mask, uint64_t key, uint32_t slot) {
#pragma unroll 1
    for (int probes = 0; probes < 16; probes++) {
        const uint32_t a = keys_addr + slot * 8u;
        const uint64_t k = lds64(a);
        if (k == key) return (int)slot;
        if (k == EMPTY_KEY) {
            const uint64_t old = atoms_cas64(a, EMPTY_KEY, key);
            if (old == EMPTY_KEY || old == key) return (int)slot;
        }
        slot = (slot + 1) & cap_mask;
    }
    return -1;
}

// `int32 column <cmp> constant` on the raw 32-bit values when the constant fits: no widening
__device__ __forceinline__ uint32_t term_mask_i32(int cmp, int32_t y, const uint32_t (&r)[8]) {
    uint32_t m = 0;
    switch (cmp) {
        case BK_FT_EQ:
#pragma unroll
            for (int j = 0; j < 4; j++) m |= ((int32_t)r[j] == y ? 1u : 0u) << j;
            break;
        case BK_FT_NE:
#pragma unroll
            for (int j = 0; j < 4; j++) m |= ((int32_t)r[j] != y ? 1u : 0u) << j;
            break;
        case BK_FT_LT:
#pragma unroll
            for (int j = 0; j < 4; j++) m |= ((int32_t)r[j] < y ? 1u : 0u) << j;
            break;
        case BK_FT_LE:
#pragma unroll
            for (int j = 0; j < 4; j++) m |= ((int32_t)r[j] <= y ? 1u : 0u) << j;
            break;
        case BK_FT_GT:
#pragma unroll
            for (int j = 0; j < 4; j++) m |= ((int32_t)r[j] > y ? 1u : 0u) << j;
            break;
        default:
#pragma unroll
            for (int j = 0; j < 4; j++) m |= ((int32_t)r[j] >= y ? 1u : 0u) << j;
            break;
    }
    return m;
}

// ------------------------------------------------------------------------------------------
// GROUP BY one column
// ------------------------------------------------------------------------------------------
template <int NP, int NA>
__global__ void __launch_bounds__(DIRECT_THREADS, 1) k_agg_group_direct(const __grid_constant__ AggArgs a) {
    constexpr int NS = NP + 1 + NA;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const AggPlan& ap = a.plan;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lane_lt = (1u << lane) - 1u;
    const bool use_smem = a.smem_cap_log2 > 0;
    const int kw = ap.n_keyw;                                  // 1 or 2
    const bool sentinel = use_smem && a.smem_sentinel != 0;    // kw == 1: keys double as slot state
    SmemTable st{};
    size_t table_bytes = 0;
    if (use_smem) {
        st = smem_table_init(smem_raw, a);
        table_bytes = (((size_t)(a.smem_keyw + a.n_smem_lanes) * 8 + 4) << a.smem_cap_log2);
    }
    // per-warp queue: [key words kw x QCAP][values NA x QCAP][null bits QCAP]
    const size_t qwords = (size_t)(kw + NA) * QCAP;
    uint64_t* qbase = (uint64_t*)(smem_raw + ((table_bytes + 15) & ~(size_t)15)) + (size_t)warp * (qwords + QCAP / 8);
    const uint32_t qkey = smem_addr(qbase);
    const uint32_t qval = qkey + (uint32_t)kw * QCAP * 8u;
    const uint32_t qnull = qkey + (uint32_t)qwords * 8u;
    const uint64_t kmask = ap.key_bits[0] >= 64 ? ~0ull : ((1ull << ap.key_bits[0]) - 1ull);
    const int null_word = ap.key_null_word[0] == 0xFF ? 0 : ap.key_null_word[0];
    const uint64_t null_bit = 1ull << ap.key_null_shift[0];
    // everything the loops need from the descriptors, resolved once into registers
    uint32_t sf[NS];
#pragma unroll
    for (int s = 0; s < NS; s++) sf[s] = slot_flags(a.cols[s]);
    const bool key_nullable = (sf[NP] & SF_HASV) != 0;
    const bool key32 = !(sf[NP] & (SF_IS8 | SF_SPECIAL));      // 4-byte integer key: its word is the raw value
    bool any_vnull = false;
#pragma unroll
    for (int s = 0; s < NA; s++) any_vnull = any_vnull || (sf[NP + 1 + s] & SF_HASV);
    bool term32[NP > 0 ? NP : 1]; int32_t term_c32[NP > 0 ? NP : 1];
#pragma unroll
    for (int t = 0; t < NP; t++) {  // int32 column against a constant that fits int32: compare raw values
        const DirectTerm tm = a.direct.term[t];
        const int64_t c = (int64_t)tm.cbits;
        term32[t] = a.cols[t].stype == ST_I32 && !(sf[t] & SF_SPECIAL) && tm.vclass == VC_I64 && c >= -2147483648ll && c <= 2147483647ll;
        term_c32[t] = (int32_t)c;
    }
    const uint32_t tcap = st.cap_mask + 1;
    const uint32_t keys_addr = smem_addr(st.keys), lanes_addr = smem_addr(st.lanes);
    const int hash_shift = 32 - a.smem_cap_log2;
    bool simple = use_smem;            // every value column feeds at most one ADD lane of its own class
    uint32_t acc_addr[NA > 0 ? NA : 1], cnt_addr[NA > 0 ? NA : 1]; bool acc_f64[NA > 0 ? NA : 1];
#pragma unroll
    for (int s = 0; s < NA; s++) {
        const ValOps vo = a.vops[s];
        acc_addr[s] = 0; cnt_addr[s] = 0; acc_f64[s] = false;
        if (vo.n_ops > 1) simple = false;
        if (vo.n_ops == 1) {
            if (!(vo.op[0] == LN_ADD_F64 || vo.op[0] == LN_ADD_I64) || (vo.lane_class[0] == VC_F64) != (vo.arg_class == VC_F64)) simple = false;
            acc_addr[s] = lanes_addr + (uint32_t)vo.smem_lane[0] * tcap * 8u; acc_f64[s] = vo.op[0] == LN_ADD_F64;
        }
        if (vo.cnt_smem != 0xFF) cnt_addr[s] = lanes_addr + (uint32_t)vo.cnt_smem * tcap * 8u;
    }
    uint32_t passed = 0;
    const int64_t nquads = a.nrows >> 2;  // full quads; the ragged rows follow the main loop
    const int64_t stride = (int64_t)gridDim.x * DIRECT_THREADS;
    int64_t q0 = (int64_t)blockIdx.x * DIRECT_THREADS + warp * 32;
    RawQuad nxt[NS];
    if (q0 + lane < nquads) {
#pragma unroll
        for (int s = 0; s < NS; s++) raw_quad_load(a.cols[s], sf[s], q0 + lane, nxt[s]);
    }
    // all lanes of a warp run the same number of iterations (the queue is warp-collective)
#pragma unroll 1
    for (; q0 < nquads; q0 += stride) {
        const int64_t q = q0 + lane;
        uint64_t kv[4]; uint32_t knm = 0;
        uint64_t vv[NA > 0 ? NA : 1][4]; uint32_t vnull[4] = {0, 0, 0, 0};
        uint32_t pass = 0;
        if (q < nquads) {
            pass = 0xFu;
#pragma unroll
            for (int t = 0; t < NP; t++) {
                if (term32[t]) pass &= term_mask_i32(a.direct.term[t].cmp, term_c32[t], nxt[t].r);
                else {
                    uint64_t pv[4];
                    raw_quad_decode(nxt[t], sf[t], a.cols[t], pv);
                    pass &= term_mask(a.direct.term[t], pv);
                }
                pass &= ~nxt[t].nm;  // NULL or false drops the row
            }
            if (key32) {
#pragma unroll
                for (int j = 0; j < 4; j++) kv[j] = nxt[NP].r[j];
            } else raw_quad_decode(nxt[NP], sf[NP], a.cols[NP], kv);
            knm = nxt[NP].nm;
#pragma unroll
            for (int s = 0; s < NA; s++) {
                raw_quad_decode(nxt[NP + 1 + s], sf[NP + 1 + s], a.cols[NP + 1 + s], vv[s]);
                if (any_vnull) {
#pragma unroll
                    for (int j = 0; j < 4; j++) vnull[j] |= ((nxt[NP + 1 + s].nm >> j) & 1u) << s;
                }
            }
        }
        // prefetch the next iteration's columns: they stay in flight while the queue is drained
        if (q + stride < nquads) {
#pragma unroll
            for (int s = 0; s < NS; s++) raw_quad_load(a.cols[s], sf[s], q + stride, nxt[s]);
        }
        // ---- compact the surviving rows of this warp into its queue: one ballot per row position ----
        uint32_t bal[4];
#pragma unroll
        for (int j = 0; j < 4; j++) bal[j] = __ballot_sync(0xFFFFFFFFu, (pass >> j) & 1u);
        int total = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if ((pass >> j) & 1u) {
                const uint32_t pos = (uint32_t)(total + __popc(bal[j] & lane_lt));
                uint64_t kword = kv[j] & kmask;
                if (key_nullable && ((knm >> j) & 1u)) {
                    kword = null_word == 0 ? null_bit : 0ull;
                    if (kw == 2) sts64(qkey + (QCAP + pos) * 8u, null_word == 1 ? null_bit : 0ull);
                } else if (kw == 2) sts64(qkey + (QCAP + pos) * 8u, 0ull);
                sts64(qkey + pos * 8u, kword);
#pragma unroll
                for (int s = 0; s < NA; s++) sts64(qval + (s * QCAP + pos) * 8u, vv[s][j]);
                if (any_vnull) sts8(qnull + pos, vnull[j]);
            }
            total += __popc(bal[j]);
        }
        passed += __popc(pass);
        __syncwarp();
        // ---- drain: every lane takes queue entries, full warps regardless of selectivity ----
        // (warp-uniform trip count: lanes beyond the tail idle inside the iteration, so the warp is
        //  converged again when it returns to the load / filter / ballot code)
#pragma unroll 1
        for (int e0 = 0; e0 < total; e0 += 32) {
            const int e = e0 + lane;
            if (e >= total) continue;
            const uint64_t k0 = lds64(qkey + e * 8u);
            const uint32_t nb = any_vnull ? lds8(qnull + e) : 0u;
            int slot = -1;
            if (sentinel) {  // Fibonacci hashing: consecutive keys land in well separated slots
                const uint32_t h = ((uint32_t)k0 ^ (uint32_t)(k0 >> 32)) * 0x9E3779B1u;
                if (k0 != EMPTY_KEY) slot = smem32_upsert1(keys_addr, st.cap_mask, k0, h >> hash_shift);
            } else if (use_smem) {
                uint64_t key[2] = {k0, lds64(qkey + (QCAP + e) * 8u)};
                slot = table_upsert<true, 2>(st.state, st.keys, st.cap_mask, key, 2, hash_key(key, 2) >> 7, 16, nullptr);
            }
            if (slot >= 0) {
                reds_inc32(lanes_addr + slot * 8u);  // lane 0 = row count (< 2^32 rows per CTA and launch)
                if (simple) {
#pragma unroll
                    for (int s = 0; s < NA; s++) {
                        if ((nb >> s) & 1u) continue;
                        if (cnt_addr[s]) reds_inc32(cnt_addr[s] + slot * 8u);
                        if (acc_addr[s]) {
                            const uint64_t v = lds64(qval + (s * QCAP + e) * 8u);
                            if (acc_f64[s]) smem32_add_f64(acc_addr[s] + slot * 8u, bits_f64(v)); else smem32_add_u64(acc_addr[s] + slot * 8u, v);
                        }
                    }
                } else {
                    uint64_t vals[NA > 0 ? NA : 1];
#pragma unroll
                    for (int s = 0; s < NA; s++) vals[s] = lds64(qval + (s * QCAP + e) * 8u);
                    smem_update_row_generic<NA>(a, st.lanes, tcap, slot, vals, nb);
                }
            } else {
                uint64_t key[2] = {k0, kw == 2 ? lds64(qkey + (QCAP + e) * 8u) : 0ull};
                uint64_t vals[NA > 0 ? NA : 1];
#pragma unroll
                for (int s = 0; s < NA; s++) vals[s] = lds64(qval + (s * QCAP + e) * 8u);
                global_update_row<NA>(a, key, vals, nb);
            }
        }
        __syncwarp();
    }
    if (use_smem) smem_table_flush(st, a);
    if (blockIdx.x == 0 && threadIdx.x < (a.nrows & 3)) passed += direct_tail_row<NP, NA>(a, (a.nrows & ~(int64_t)3) + threadIdx.x);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) passed += __shfl_xor_sync(0xFFFFFFFFu, passed, d);
    if (lane == 0 && passed) atomicAdd((unsigned long long*)a.rows_passed, (unsigned long long)passed);
}


// ------------------------------------------------------------------------------------------
// FX — double sums as fixed-point limbs (the lean kernel's default for SUM / AVG over DOUBLE columns)
// Why: sm_90a's shared memory has native atomics for 32-bit integers only; a double add is LDS -> DADD -> ATOMS.CAS in a loop, and a
// pass of 32 random group slots through `RED.u32 + LDS.128 + ATOMS.CAS.128` costs more SM cycles than `RED.u32 + 2 x (ATOMS.ADD + RED)`,
// and more still with few groups, where the compare-and-swap retries (scripts/mb/mb_atoms.cu measures both).
// How: per CTA and value column a power-of-two scale 2^F is chosen from a sample of the batch (640 rows spread over the whole column),
// so that the largest value seen has M - 3 significant bits above the quantum; M = 62 - ceil(log2(rows this CTA can add)) keeps the
// 64-bit sum of one slot from overflowing whatever the key distribution.  A value x becomes y = x * 2^F (exact) and takes one of
//   main  2^(M-15) <= |y| < 2^M : round(y) added to the slot's {mid, hi} limbs, ATOMS.ADD.32 with the carry folded into a RED.32;
//                                 relative rounding error per value <= 2^-(M-14), i.e. M - 14 significant bits; M falls with the rows
//                                 one CTA adds: on 132 SMs one batch of 100M rows has M = 42 (28 bits, 3.7e-9), of 300M rows M = 40
//                                 (26 bits, 1.5e-8); typically 1e-12,
//   fine  2^(M-47) <= |y| < 2^(M-15) : round(y * 2^32) added to {ext, mid, hi} (three limbs, same per-value precision),
//   zero  nothing to add,
//   else  (beyond the sampled range, denormal, Inf, NaN): an exact double add into the global table.
// A CTA's partial sum of a group is therefore the exact sum of values rounded to at least M-14 significant bits each — it does not
// depend on the order in which the atomics land — with an error <= 2^-(M-14) relative to sum(|x|) in the worst case (2^-28 at M = 42,
// 2^-26 at M = 40), against north_star's 1e-6 (tests/sum_bounds.py states the whole bound, tests/test_gpu_double_sums.py measures it).  At flush time the limbs become one double per lane and the table is merged as before (the CTAs' partial sums meet as doubles
// in the global table: RED.E.ADD.F64).
// (AggFnCall::update's `add` is a sequential double add, agg_fn_call.cpp:496-555; any parallel order already differs from it in the
// last bits.)
// ------------------------------------------------------------------------------------------
// (out of line although the call costs 24 bytes of spills: inlined, this rare path makes the loop outgrow the instruction cache)
static __device__ __noinline__ void global_add_f64(const AggArgs& a, uint64_t k0, int glob_lane, double x) {
    const AggPlan& ap = a.plan;
    const GroupTable& gt = a.gt;
    const uint32_t gcap = gt.cap_mask + 1;
    uint64_t key[MAX_KEYW];
    key[0] = k0;
    for (int w = 1; w < MAX_KEYW; w++) key[w] = 0ull;
    const int slot = table_upsert<false, 0>(gt.state, gt.keys, gt.cap_mask, key, ap.n_keyw, ap.n_keyw == 1 ? hash_key1(key[0]) : hash_key(key, ap.n_keyw), (int)gcap, gt.n_groups);
    if (slot < 0) { atomicExch(gt.overflow, 1u); return; }
    lane_atomic<false>(LN_ADD_F64, gt.lanes + (size_t)glob_lane * gcap + slot, f64_bits(x));
    atomicAdd(gt.n_groups + GT_FX_EXACT, 1u);   // values that took this path: when they are many the host stops choosing FX for this plan (agg.cu)
}
__device__ __forceinline__ void reds_add32(uint32_t a, uint32_t v) { asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
// one value into the fixed-point limbs of `slot`: word = shared address of the slot's {mid, hi} pair, ext = of its low-extension limb
__device__ __forceinline__ void fx_add(const AggArgs& a, uint32_t word, uint32_t ext, double scale, uint32_t fx_lo, uint64_t k0, int glob_lane, uint64_t vbits) {
    uint32_t lo; uint64_t up;
    const int kind = fx_split(bits_f64(vbits), scale, fx_lo, lo, up);
    if (kind == FX_MAIN) {
        const uint32_t old = atoms_add32(word, lo);
        const uint32_t h = (uint32_t)up + ((old + lo) < old ? 1u : 0u);
        if (h) reds_add32(word + 4u, h);
    } else if (kind == FX_FINE) {
        const uint32_t old = atoms_add32(ext, lo);
        const uint64_t t = up + ((old + lo) < old ? 1u : 0u);   // sign-extended upper part + carry
        const uint32_t m = (uint32_t)t;
        const uint32_t old2 = atoms_add32(word, m);
        const uint32_t h = (uint32_t)(t >> 32) + ((old2 + m) < old2 ? 1u : 0u);
        if (h) reds_add32(word + 4u, h);
    } else if (kind == FX_EXACT) global_add_f64(a, k0, glob_lane, bits_f64(vbits));
}

// ------------------------------------------------------------------------------------------
// GROUP BY one column, LEAN shape — what the headline query (config C2/C4) and most star-schema
// aggregations look like: no NULLs in this batch, every predicate term is `int32 column <cmp> int32
// constant`, the key is a 4- or 8-byte integer column, every value column is 8 bytes wide and feeds
// exactly one SUM lane (double or int64) — COUNT(*) and AVG ride on the row count.  With all of that
// fixed the hot loop has no descriptor interpretation left in it.  Everything else takes
// k_agg_group_direct above (same results, more instructions per row).
// ------------------------------------------------------------------------------------------
// NULLS: predicate / value columns may carry validity bitmaps (a NULL predicate operand drops the row, a NULL value skips that
// aggregate: its sum gets +0 and its non-NULL counter no increment); the key column stays NULL-free in this kernel.
// MM: value columns may feed MIN / MAX lanes (LDS -> compare -> ATOMS.CAS.64 only when the row improves the extreme: after the
// first rows of a group that is one LDS per row) and up to three lanes each (SUM + MIN + MAX over one column).
// FX: double sums as fixed-point limbs updated with native 32-bit shared atomics (see above).
template <int NP, int NA, bool JOIN, bool NULLS = false, bool MM = false, bool FX = false>
__global__ void __launch_bounds__(LEAN_THREADS, 1) k_agg_group_lean(const __grid_constant__ AggArgs a) {
    constexpr int NS = NP + 1 + NA;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const AggPlan& ap = a.plan;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lane_lt = (1u << lane) - 1u;
    SmemTable st = smem_table_init(smem_raw, a);
    const size_t table_bytes = (((size_t)(1 + a.n_smem_lanes) * 8 + 4) << a.smem_cap_log2);
    // per-warp queue: a ring of LEAN_QCAP entries [key][values NA][null bytes].  Only FULL passes of 32 entries are drained;
    // the < 32 left over wait for the next iteration's survivors (at 50 % selectivity 64 +- 6 rows survive per iteration:
    // draining whatever arrived costs 2.5 passes on average, the last one nearly empty; carrying the remainder costs 2.0)
    constexpr uint32_t LQ = LEAN_QCAP;
    const size_t qwords = (size_t)(1 + NA) * LQ;
    // (each warp's ring starts on a 128-byte boundary: a pass of 32 consecutive 8-byte entries is then exactly two wavefronts)
    uint64_t* qbase = (uint64_t*)(smem_raw + ((table_bytes + 127) & ~(size_t)127)) + (size_t)warp * ((qwords + LQ / 8 + 15) & ~(size_t)15);
    const uint32_t qkey = smem_addr(qbase);
    const uint32_t qval = qkey + LQ * 8u;
    const uint32_t qnull = qkey + (uint32_t)qwords * 8u;   // NULLS: one byte of per-value NULL bits per queue entry
    const uint64_t kmask = ap.key_bits[0] >= 64 ? ~0ull : ((1ull << ap.key_bits[0]) - 1ull);
    const bool key8 = a.cols[NP].stype == ST_I64 || a.cols[NP].stype == ST_U64;
    const uint32_t cap_mask = st.cap_mask, tcap = st.cap_mask + 1;
    const uint32_t keys_addr = smem_addr(st.keys), lanes_addr = smem_addr(st.lanes);
    const int hash_shift = 32 - a.smem_cap_log2;
    int tcmp[NP > 0 ? NP : 1]; int32_t tconst[NP > 0 ? NP : 1];
    const uint8_t* tptr[NP > 0 ? NP : 1];
#pragma unroll
    for (int t = 0; t < NP; t++) { tcmp[t] = a.direct.term[t].cmp; tconst[t] = (int32_t)(int64_t)a.direct.term[t].cbits; tptr[t] = (const uint8_t*)a.cols[t].values; }
    const uint8_t* kptr = (const uint8_t*)a.cols[NP].values;
    const uint8_t* vptr[NA > 0 ? NA : 1]; uint32_t acc_addr[NA > 0 ? NA : 1]; bool acc_f64[NA > 0 ? NA : 1];
#pragma unroll
    for (int s = 0; s < NA; s++) {
        vptr[s] = (const uint8_t*)a.cols[NP + 1 + s].values;
        const uint32_t sl = a.vops[s].smem_lane[0];                              // paired layout: word ((sl/2)*cap + slot)*2 + sl%2
        acc_addr[s] = lanes_addr + ((sl >> 1) * tcap * 2u + (sl & 1u)) * 8u;
        acc_f64[s] = a.vops[s].op[0] == LN_ADD_F64;
    }
    const uint8_t* valid[NS]; uint32_t cnt_addr[NA > 0 ? NA : 1];
    if (NULLS) {
#pragma unroll
        for (int t = 0; t < NP; t++) valid[t] = a.cols[t].validity;
        valid[NP] = nullptr;
#pragma unroll
        for (int s = 0; s < NA; s++) {
            valid[NP + 1 + s] = a.cols[NP + 1 + s].validity;
            const uint32_t cl = a.vops[s].cnt_smem;   // shared lane of the non-NULL counter (0xFF: the column has no NULLs in this batch)
            cnt_addr[s] = cl == 0xFF ? 0u : lanes_addr + ((cl >> 1) * tcap * 2u + (cl & 1u)) * 8u;
        }
    }
    uint32_t nmask = 0;   // NULLS: 4 NULL bits per column for the quad held in the load registers
    // 128-bit shared CAS shape: {sumA, sumB} — value columns 0 and 1 both feed one double sum and share a 16-byte word.
    // (Fusing {row count, sum} into one CAS.128 for a single double sum is not used: the native 32-bit
    //  reduction is cheaper than widening the compare-and-swap.)
    const bool pair2 = NA >= 2 && acc_f64[0] && acc_f64[NA > 1 ? 1 : 0] && a.vops[0].smem_lane[0] == 2 && a.vops[NA > 1 ? 1 : 0].smem_lane[0] == 3 &&
                       (!MM || (a.vops[0].n_ops == 1 && a.vops[NA > 1 ? 1 : 0].n_ops == 1));
    uint32_t passed = 0;
    const int64_t nquads = a.nrows >> 2;
    const int64_t stride = (int64_t)gridDim.x * LEAN_THREADS;
    // ---- FX: per-CTA scale of every double sum, from a sample of 640 rows spread over the whole batch ----
    double fx_scale[NA > 0 ? NA : 1]; uint32_t fx_lo = 0, fx_ext = 0;
    __shared__ uint32_t fx_emax[4];
    __shared__ int32_t fx_F[4];
    if constexpr (FX) {
        fx_ext = smem_addr(smem_raw) + a.fx_ext_off;
        if (threadIdx.x < 4) fx_emax[threadIdx.x] = 0u;
        for (uint32_t i = threadIdx.x; i < (uint32_t)NA * tcap; i += LEAN_THREADS) sts32(fx_ext + i * 4u, 0u);
        for (uint32_t i = threadIdx.x; i < tcap; i += LEAN_THREADS) {   // the limbs start from integer 0, not from the lane's -0.0
#pragma unroll
            for (int s = 0; s < NA; s++) if (acc_f64[s]) sts64(acc_addr[s] + i * 16u, 0ull);
        }
        __syncthreads();
        const int64_t srow = (int64_t)((uint64_t)(blockIdx.x + (uint64_t)threadIdx.x * gridDim.x) * (uint64_t)a.nrows / ((uint64_t)gridDim.x * LEAN_THREADS));
#pragma unroll
        for (int s = 0; s < NA; s++) {
            if (!acc_f64[s]) continue;
            uint32_t e = (uint32_t)(__ldg((const unsigned long long*)vptr[s] + srow) >> 52) & 0x7FFu;
            if (e == 0x7FFu) e = 0u;   // Inf / NaN say nothing about the scale (they take the exact path anyway)
            e = __reduce_max_sync(0xFFFFFFFFu, e);
            if (lane == 0) atomicMax(&fx_emax[s], e);
        }
        __syncthreads();
        const uint64_t rows_cta = (uint64_t)((nquads + stride - 1) / stride) * (LEAN_THREADS * 4u) + 4u;   // rows this CTA can add to one slot
        const int M = fx_magnitude_bits(rows_cta | FX_MIN_ROWS);   // <= FX_MAX_M
        fx_lo = fx_floor_exp(M);
#pragma unroll
        for (int s = 0; s < NA; s++) {
            const int F = fx_scale_exp(M, fx_emax[s]);
            fx_scale[s] = fx_pow2(F);
            if (threadIdx.x == 0) fx_F[s] = F;
        }
    }
    int64_t q0 = (int64_t)blockIdx.x * LEAN_THREADS + warp * 32;
    uint32_t pr[NP > 0 ? NP : 1][4]; uint32_t kr[8]; uint64_t vr[NA > 0 ? NA : 1][4];
    auto issue_loads = [&](int64_t q) {
#pragma unroll
        for (int t = 0; t < NP; t++) { const U32x4 r = ldg128_u32(tptr[t] + q * 16);
#pragma unroll
            for (int j = 0; j < 4; j++) pr[t][j] = r.v[j]; }
        if (key8) { const U32x8 r = ldg256_u32(kptr + q * 32);
#pragma unroll
            for (int j = 0; j < 8; j++) kr[j] = r.v[j]; }
        else { const U32x4 r = ldg128_u32(kptr + q * 16);
#pragma unroll
            for (int j = 0; j < 4; j++) kr[j] = r.v[j]; }
#pragma unroll
        for (int s = 0; s < NA; s++) { const U64x4 r = ldg256_u64(vptr[s] + q * 32);
#pragma unroll
            for (int j = 0; j < 4; j++) vr[s][j] = r.v[j]; }
        if (NULLS) {
            nmask = 0;
#pragma unroll
            for (int c = 0; c < NS; c++)
                if (c != NP && valid[c]) nmask |= ((~((uint32_t)__ldg(valid[c] + (q >> 1)) >> ((q & 1) * 4))) & 0xFu) << (4 * c);
        }
    };
    auto fx_finish = [&]() {   // FX: the limbs of every slot become the double the flush expects in the lane's word
        if constexpr (FX) {
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < tcap; i += LEAN_THREADS) {
#pragma unroll
                for (int s = 0; s < NA; s++) {
                    if (!acc_f64[s]) continue;
                    const uint32_t word = acc_addr[s] + i * 16u;
                    const long long top = (long long)lds64(word);                       // {mid, hi}: the sum in units of 2^-F
                    const uint32_t ext = lds32(fx_ext + ((uint32_t)s * tcap + i) * 4u);   // units of 2^-(F+32)
                    const double sum = fx_combine(top, ext, fx_F[s]);
                    sts64(word, f64_bits(sum));
                }
            }
        }
    };
    if (q0 + lane < nquads) issue_loads(q0 + lane);
    uint32_t qhead = 0, qcount = 0;   // warp-uniform: ring start (a multiple of 32) and entries waiting in it
#pragma unroll 1
    for (;;) {
        const bool last = q0 >= nquads;   // (warp-uniform) one extra trip drains what is left in the ring
        uint32_t total = qcount;
        if (!last) {
        const int64_t q = q0 + lane;
        uint32_t pass = 0;
        if (q < nquads) {
            pass = 0xFu;
#pragma unroll
            for (int t = 0; t < NP; t++) {
                uint32_t r8[8];
#pragma unroll
                for (int j = 0; j < 4; j++) r8[j] = pr[t][j];
                pass &= term_mask_i32(tcmp[t], tconst[t], r8);
                if (NULLS) pass &= ~(nmask >> (4 * t));
            }
        }
        const uint32_t vnull = NULLS ? nmask >> (4 * (NP + 1)) : 0u;   // per value column s: bits [4s, 4s+4) = rows j
        if (JOIN) {
            // K4 fused: the foreign keys of the surviving rows become the dimension attribute the query groups by; the
            // four lookups of a lane fly together, rows without a partner leave the mask (inner join)
            const JoinProbe& jp = a.jp;
            uint32_t g[4]; uint32_t hit = 0;
            if (jp.mode == 1) {
                uint64_t off[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint64_t img = jp.key_signed ? (uint64_t)(int64_t)(int32_t)kr[j] : (uint64_t)kr[j];
                    off[j] = (img ^ jp.bias) - jp.dense_min;
                    g[j] = 0;
                    if (((pass >> j) & 1u) && off[j] < jp.dense_size) { g[j] = __ldg(jp.attr + off[j]); hit |= 1u << j; }
                }
                if (jp.present) {
                    uint32_t pr4[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) pr4[j] = ((hit >> j) & 1u) ? __ldg(jp.present + off[j]) : 0xFFFFFFFFu;
#pragma unroll
                    for (int j = 0; j < 4; j++) if (pr4[j] == 0xFFFFFFFFu) hit &= ~(1u << j);
                }
            } else {
                uint32_t slot[4]; uint64_t e[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    slot[j] = (kr[j] * 0x9E3779B1u) & jp.packed_mask;
                    e[j] = ((pass >> j) & 1u) ? __ldg((const unsigned long long*)(jp.packed + slot[j])) : ~0ull;
                }
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    g[j] = 0;
                    while (e[j] != ~0ull) {
                        if ((uint32_t)(e[j] >> 32) == kr[j]) { g[j] = (uint32_t)e[j]; hit |= 1u << j; break; }
                        slot[j] = (slot[j] + 1) & jp.packed_mask;
                        e[j] = __ldg((const unsigned long long*)(jp.packed + slot[j]));
                    }
                }
            }
            pass &= hit;
#pragma unroll
            for (int j = 0; j < 4; j++) kr[j] = g[j];
        }
        // compact the surviving rows of this warp into its queue (straight from the load registers) ...
        uint32_t bal[4];
#pragma unroll
        for (int j = 0; j < 4; j++) bal[j] = __ballot_sync(0xFFFFFFFFu, (pass >> j) & 1u);
        uint32_t fresh = 0;
        const uint32_t tail = qhead + qcount;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if ((pass >> j) & 1u) {
                uint32_t pos = tail + fresh + (uint32_t)__popc(bal[j] & lane_lt);
                if (NP > 0) pos -= pos >= LQ ? LQ : 0u;   // (no filter: nothing is ever carried, positions stay below 128)
                sts64(qkey + pos * 8u, key8 ? ((uint64_t)kr[2 * j] | ((uint64_t)kr[2 * j + 1] << 32)) : ((uint64_t)kr[j] & kmask));
#pragma unroll
                for (int s = 0; s < NA; s++) sts64(qval + (s * LQ + pos) * 8u, vr[s][j]);
                if (NULLS) {
                    uint32_t nb = 0;
#pragma unroll
                    for (int s = 0; s < NA; s++) nb |= ((vnull >> (4 * s + j)) & 1u) << s;
                    sts8(qnull + pos, nb);
                }
            }
            fresh += __popc(bal[j]);
        }
        total += fresh;
        // ... then reuse those registers for the next iteration's columns: they fly while the queue drains
        if (q + stride < nquads) issue_loads(q + stride);
        passed += __popc(pass);
        }
        __syncwarp();
        // (without a filter every iteration brings exactly four full passes: nothing to carry, the ring stays at 0)
        const uint32_t limit = (last || NP == 0) ? total : (total & ~31u);
        // (one entry per lane: a two-entries-per-lane variant needs more registers and leaves more
        //  lanes idle in the last pass)
#pragma unroll 1
        for (uint32_t e0 = 0; e0 < limit; e0 += 32) {
            if (e0 + lane >= limit) continue;   // (only the final trip has a ragged pass)
            uint32_t e = qhead + e0 + lane;
            if (NP > 0) e -= e >= LQ ? LQ : 0u;
            const uint64_t k0 = lds64(qkey + e * 8u);
            uint64_t v[NA > 0 ? NA : 1];
#pragma unroll
            for (int s = 0; s < NA; s++) v[s] = lds64(qval + (s * LQ + e) * 8u);
            uint32_t nb = 0;
            if (NULLS) {
                nb = lds8(qnull + e);
#pragma unroll
                for (int s = 0; s < NA; s++) if ((nb >> s) & 1u) v[s] = acc_f64[s] ? 0x8000000000000000ull : 0ull;   // 0 / -0.0 leaves the sum unchanged
            }
            const uint32_t h = ((uint32_t)k0 ^ (uint32_t)(k0 >> 32)) * 0x9E3779B1u;
            int slot = -1;
            if (k0 != EMPTY_KEY) slot = smem32_upsert1(keys_addr, cap_mask, k0, h >> hash_shift);
            if (slot >= 0) {
                if constexpr (FX) {   // native 32-bit atomics only: row count, then two (rarely three) limbs per double sum
                    reds_inc32(lanes_addr + slot * 16u);
#pragma unroll
                    for (int s = 0; s < NA; s++) {
                        if (acc_f64[s]) fx_add(a, acc_addr[s] + slot * 16u, fx_ext + ((uint32_t)s * tcap + slot) * 4u, fx_scale[s], fx_lo, k0, a.vops[s].glob_lane[0], v[s]);
                        else smem32_add_u64(acc_addr[s] + slot * 16u, v[s]);
                    }
                } else {
                    reds_inc32(lanes_addr + slot * 16u);   // pair 0, half 0 = row count
                    if (NULLS) {
#pragma unroll
                        for (int s = 0; s < NA; s++) if (cnt_addr[s] && !((nb >> s) & 1u)) reds_inc32(cnt_addr[s] + slot * 16u);
                    }
                    int first = 0;
                    if (pair2) {   // {sumA, sumB}: both double sums of the group move in one ATOMS.CAS.128
                        const uint32_t addr = acc_addr[0] + slot * 16u;
                        uint64_t c0, c1;
                        lds128(addr, c0, c1);
                        for (;;) {
                            uint64_t p0, p1;
                            atoms_cas128(addr, c0, c1, f64_bits(bits_f64(c0) + bits_f64(v[0])), f64_bits(bits_f64(c1) + bits_f64(v[NA > 1 ? 1 : 0])), p0, p1);
                            if (p0 == c0 && p1 == c1) break;
                            c0 = p0; c1 = p1;
                        }
                        first = 2;
                    }
#pragma unroll
                    for (int s = 0; s < NA; s++) {
                        if (s < first) continue;
                        if (MM) {
                            if (NULLS && ((nb >> s) & 1u)) continue;   // a NULL input touches no lane
                            const int nops = a.vops[s].n_ops;
#pragma unroll 1
                            for (int k = 0; k < nops; k++) {
                                const int op = a.vops[s].op[k];
                                const uint32_t sl = a.vops[s].smem_lane[k];
                                const uint32_t addr = lanes_addr + ((sl >> 1) * tcap * 2u + (sl & 1u)) * 8u + slot * 16u;
                                if (op == LN_ADD_F64) smem32_add_f64(addr, bits_f64(v[s]));
                                else if (op == LN_ADD_I64) smem32_add_u64(addr, v[s]);
                                else smem32_minmax(addr, op, v[s]);
                            }
                        }
                        else if (acc_f64[s]) smem32_add_f64(acc_addr[s] + slot * 16u, bits_f64(v[s])); else smem32_add_u64(acc_addr[s] + slot * 16u, v[s]);
                    }
                }
            } else {   // rare: re-read the entry from the queue so that v[] never needs an address (no local-memory copy per pass)
                uint64_t key[2] = {k0, 0ull};
                uint64_t gv[NA > 0 ? NA : 1];
#pragma unroll
                for (int s = 0; s < NA; s++) gv[s] = lds64(qval + (s * LQ + e) * 8u);
                global_update_row<NA>(a, key, gv, nb);
            }
        }
        if (NP > 0) { qhead = (qhead + limit) % LQ; qcount = total - limit; }
        __syncwarp();
        if (last) break;
        q0 += stride;
    }
    fx_finish();
    smem_table_flush(st, a);
    if (blockIdx.x == 0 && threadIdx.x < (a.nrows & 3)) passed += direct_tail_row<NP, NA, JOIN>(a, (a.nrows & ~(int64_t)3) + threadIdx.x);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) passed += __shfl_xor_sync(0xFFFFFFFFu, passed, d);
    if (lane == 0 && passed) atomicAdd((unsigned long long*)a.rows_passed, (unsigned long long)passed);
    if (a.fused_out) fused_extract(a);
}

// ------------------------------------------------------------------------------------------
// no GROUP BY: accumulate in registers (per value column up to 3 lane operations), warp shuffle
// reduction, one set of global atomics per warp
// ------------------------------------------------------------------------------------------
template <int NP, int NA>
__global__ void __launch_bounds__(DIRECT_THREADS, NA == 0 ? 2 : 1) k_agg_scalar_direct(const __grid_constant__ AggArgs a) {   // COUNT(*) only: two CTAs per SM
    constexpr int NS = NP + NA;
    const int lane = threadIdx.x & 31;
    uint64_t rows = 0;
    uint64_t acc[NA > 0 ? NA : 1][3], cnt[NA > 0 ? NA : 1];
#pragma unroll
    for (int s = 0; s < NA; s++) {
        cnt[s] = 0;
#pragma unroll
        for (int k = 0; k < 3; k++) acc[s][k] = k < a.vops[s].n_ops ? lane_identity(a.vops[s].op[k]) : 0;
    }
    uint32_t sf[NS > 0 ? NS : 1];
#pragma unroll
    for (int s = 0; s < NS; s++) sf[s] = slot_flags(a.cols[s]);
    // `int32 column <cmp> int32 constant` terms compare the loaded words directly (no 64-bit decode)
    bool term32[NP > 0 ? NP : 1]; int32_t term_c32[NP > 0 ? NP : 1];
#pragma unroll
    for (int t = 0; t < NP; t++) {
        const DirectTerm tm = a.direct.term[t];
        const int64_t c = (int64_t)tm.cbits;
        term32[t] = a.cols[t].stype == ST_I32 && !(sf[t] & SF_SPECIAL) && tm.vclass == VC_I64 && c >= -2147483648ll && c <= 2147483647ll;
        term_c32[t] = (int32_t)c;
    }
    const int64_t nquads = a.nrows >> 2;
    // U independent row quads per thread and trip: with one or two narrow columns a single 16-byte load per thread
    // leaves too few bytes in flight to cover HBM latency (132 SMs x 512 threads x 16 B = 1.1 MB)
    constexpr int U = NS <= 1 ? 4 : (NS <= 3 ? 2 : 1);
    const int64_t T = (int64_t)gridDim.x * DIRECT_THREADS;
#pragma unroll 1
    for (int64_t q0 = (int64_t)blockIdx.x * DIRECT_THREADS + threadIdx.x; q0 < nquads; q0 += T * U) {
      RawQuad rawu[U][NS > 0 ? NS : 1];
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (q0 + u * T < nquads) {
#pragma unroll
            for (int s = 0; s < NS; s++) raw_quad_load(a.cols[s], sf[s], q0 + u * T, rawu[u][s]);
        }
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (q0 + u * T >= nquads) break;
        RawQuad (&raw)[NS > 0 ? NS : 1] = rawu[u];
        uint32_t pass = 0xFu;
#pragma unroll
        for (int t = 0; t < NP; t++) {
            if (term32[t]) pass &= term_mask_i32(a.direct.term[t].cmp, term_c32[t], raw[t].r) & ~raw[t].nm;
            else {
                uint64_t pv[4];
                raw_quad_decode(raw[t], sf[t], a.cols[t], pv);
                pass &= term_mask(a.direct.term[t], pv) & ~raw[t].nm;
            }
        }
        rows += __popc(pass);
#pragma unroll
        for (int s = 0; s < NA; s++) {
            uint64_t v[4];
            raw_quad_decode(raw[NP + s], sf[NP + s], a.cols[NP + s], v);
            const uint32_t ok = pass & ~raw[NP + s].nm;
            cnt[s] += __popc(ok);
            const ValOps vo = a.vops[s];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                if (k >= vo.n_ops) break;
                const int op = vo.op[k];
                if (op == LN_ADD_F64 && vo.arg_class == VC_F64) {
                    double d = bits_f64(acc[s][k]);
#pragma unroll
                    for (int j = 0; j < 4; j++) if ((ok >> j) & 1u) d += bits_f64(v[j]);
                    acc[s][k] = f64_bits(d);
                } else if (op == LN_ADD_I64) {
#pragma unroll
                    for (int j = 0; j < 4; j++) if ((ok >> j) & 1u) acc[s][k] += v[j];
                } else acc[s][k] = combine4_generic(op, acc[s][k], v, ok, vo.arg_class, vo.lane_class[k]);
            }
        }
      }
    }
    const GroupTable& gt = a.gt;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) rows += __shfl_xor_sync(0xFFFFFFFFu, rows, d);
#pragma unroll
    for (int s = 0; s < NA; s++) {
        const ValOps vo = a.vops[s];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) cnt[s] += __shfl_xor_sync(0xFFFFFFFFu, cnt[s], d);
#pragma unroll
        for (int k = 0; k < 3; k++) {
            if (k >= vo.n_ops) break;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) acc[s][k] = lane_combine(vo.op[k], acc[s][k], __shfl_xor_sync(0xFFFFFFFFu, acc[s][k], d));
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (a.nrows & 3)) {
        const uint32_t p1 = direct_tail_row<NP, NA>(a, (a.nrows & ~(int64_t)3) + threadIdx.x);
        if (p1) atomicAdd((unsigned long long*)a.rows_passed, 1ull);
    }
    if (lane == 0) {  // the single group lives in slot 0 (capacity 1): lane l is gt.lanes[l]
        if (rows) { atomicAdd((unsigned long long*)gt.lanes, (unsigned long long)rows); atomicAdd((unsigned long long*)a.rows_passed, (unsigned long long)rows); }
#pragma unroll
        for (int s = 0; s < NA; s++) {
            const ValOps vo = a.vops[s];
            if (cnt[s] == 0) continue;
            if (vo.cnt_glob) atomicAdd((unsigned long long*)(gt.lanes + vo.cnt_glob), (unsigned long long)cnt[s]);
            for (int k = 0; k < vo.n_ops; k++) lane_atomic<false>(vo.op[k], gt.lanes + vo.glob_lane[k], acc[s][k]);
        }
    }
}

// ------------------------------------------------------------------------------------------
// Launch setup paid once per kernel: its dynamic shared-memory limit is raised only when a launch needs more than was set before, and
// its resident CTAs per SM are asked once per (device, threads, shared bytes) — the answers never change, and asking costs
// microseconds of host time on every request.
struct LaunchSetupCache {
    std::mutex mu;
    std::map<std::pair<int, const void*>, size_t> smem_set;
    std::map<std::tuple<int, const void*, int, size_t>, int> per_sm;
};
inline LaunchSetupCache& launch_setup_cache() { static LaunchSetupCache c; return c; }

// persistent grid: whole CTAs per SM x the device's SMs (132 on H100 SXM), fewer for a small batch.  `start` (optional) is recorded
// right before the launch, after the setup, so that it times the kernel alone.
template <class K>
static inline cudaError_t launch_persistent(K kernel, const AggArgs& a, size_t smem, int sm_count, int threads, cudaStream_t s, cudaEvent_t start) {
    int dev = 0, per_sm = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    {
        LaunchSetupCache& c = launch_setup_cache();
        std::lock_guard<std::mutex> g(c.mu);
        if (smem > 48 * 1024) {
            size_t& have = c.smem_set[{dev, (const void*)kernel}];
            if (smem > have) {
                if ((e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
                have = smem;
            }
        }
        const auto key = std::make_tuple(dev, (const void*)kernel, threads, smem);
        const auto it = c.per_sm.find(key);
        if (it != c.per_sm.end()) per_sm = it->second;
        else {
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
            c.per_sm[key] = per_sm;
        }
    }
    const int64_t want = ((a.nrows + 3) / 4 + threads - 1) / threads;
    const int64_t full = (int64_t)per_sm * sm_count;
    if (start) cudaEventRecord(start, s);
    kernel<<<(int)(want < full ? want : full), threads, smem, s>>>(a);
    return cudaGetLastError();
}

// the kernel select_agg_launch (agg_select.cpp) chose; exactly these instantiations of k_agg_group_lean exist
template <int NP, int NA>
static inline cudaError_t launch_direct(const AggArgs& a, AggKernel k, int sm_count, size_t smem, cudaStream_t s, cudaEvent_t start) {
    constexpr int T = LEAN_THREADS;
    switch (k) {
        case SCALAR_DIRECT: return launch_persistent(k_agg_scalar_direct<NP, NA>, a, 0, sm_count, DIRECT_THREADS, s, start);
        case GROUP_DIRECT: return launch_persistent(k_agg_group_direct<NP, NA>, a, smem, sm_count, DIRECT_THREADS, s, start);
        case LEAN: return launch_persistent(k_agg_group_lean<NP, NA, false>, a, smem, sm_count, T, s, start);
        // (one MM / NULLS instantiation serves batches with and without NULLs: without bitmaps the NULL masks are simply zero)
        case LEAN_MM: return launch_persistent(k_agg_group_lean<NP, NA, false, true, true>, a, smem, sm_count, T, s, start);
        case LEAN_NULLS: return launch_persistent(k_agg_group_lean<NP, NA, false, true>, a, smem, sm_count, T, s, start);
        case LEAN_JOIN: return launch_persistent(k_agg_group_lean<NP, NA, true>, a, smem, sm_count, T, s, start);
        case LEAN_FX:   // double sums as fixed-point limbs (native 32-bit shared atomics)
            if constexpr (NA >= 1) return launch_persistent(k_agg_group_lean<NP, NA, false, false, false, true>, a, smem, sm_count, T, s, start);
            break;
        case LEAN_FX_JOIN:
            if constexpr (NA >= 1) return launch_persistent(k_agg_group_lean<NP, NA, true, false, false, true>, a, smem, sm_count, T, s, start);
            break;
        default: break;
    }
    return cudaErrorInvalidValue;
}
template <int NP>
static inline cudaError_t launch_direct_np(const AggArgs& a, AggKernel k, int sm_count, size_t smem, cudaStream_t s, cudaEvent_t start) {
    switch (a.direct.n_vals) {
        case 0: return launch_direct<NP, 0>(a, k, sm_count, smem, s, start);
        case 1: return launch_direct<NP, 1>(a, k, sm_count, smem, s, start);
        case 2: return launch_direct<NP, 2>(a, k, sm_count, smem, s, start);
        case 3: return launch_direct<NP, 3>(a, k, sm_count, smem, s, start);
        default: return launch_direct<NP, 4>(a, k, sm_count, smem, s, start);
    }
}

}  // namespace bk

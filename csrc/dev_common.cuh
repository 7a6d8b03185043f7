// dev_common.cuh — device-side building blocks shared by the kernels: vectorised column loads
// (32 bytes per lane as two LDG.128 on sm_90a), ExprValue arithmetic on canonical 64-bit images, the open-addressed group
// table (same code for shared and global memory) and the accumulator lane operations.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "dev_types.h"
#include "../include/bkgpu_plan.h"
#include "datetime.h"

namespace bk {

// ------------------------------------------------------------------------------------------
// streaming loads.  Column data is read exactly once: bypass L1 allocation.
// ------------------------------------------------------------------------------------------
struct alignas(16) U32x4 { uint32_t v[4]; };
struct alignas(32) U32x8 { uint32_t v[8]; };
struct alignas(32) U64x4 { uint64_t v[4]; };

__device__ __forceinline__ U32x4 ldg128_u32(const void* p) {
    U32x4 r;
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
        : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]) : "l"(p));
    return r;
}
// 32 bytes per lane.  sm_90a's widest global load is 128 bits, so a 32-byte chunk is two LDG.128 issued
// back to back (both in flight before either result is used).
__device__ __forceinline__ U32x8 ldg256_u32(const void* p) {
    U32x8 r;
    asm("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
        "ld.global.nc.L1::no_allocate.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
                 : "l"(p));
    return r;
}
__device__ __forceinline__ U64x4 ldg256_u64(const void* p) {
    U64x4 r;
    asm("ld.global.nc.L1::no_allocate.v2.u64 {%0,%1}, [%4];\n\t"
        "ld.global.nc.L1::no_allocate.v2.u64 {%2,%3}, [%4+16];"
                 : "=l"(r.v[0]), "=l"(r.v[1]), "=l"(r.v[2]), "=l"(r.v[3]) : "l"(p));
    return r;
}

__device__ __forceinline__ uint64_t f64_bits(double d) { return (uint64_t)__double_as_longlong(d); }
__device__ __forceinline__ double bits_f64(uint64_t b) { return __longlong_as_double((long long)b); }

// Re-narrow a canonical image to the slot's declared type: SlotRef::get_value does
// row->get_value(...).cast_to(_col_type) (include/expr/slot_ref.h:31-40) and INT8/INT16 travel in
// 32-bit storage (src/runtime/chunk.cpp:48-53).
__device__ __forceinline__ uint64_t narrow_prim(uint64_t v, int prim) {
    switch (prim) {
        case BK_INT8: return (uint64_t)(int64_t)(int8_t)v;
        case BK_INT16: return (uint64_t)(int64_t)(int16_t)v;
        case BK_UINT8: return (uint64_t)(uint8_t)v;
        case BK_UINT16: return (uint64_t)(uint16_t)v;
        case BK_BOOL: return v != 0;
        default: return v;
    }
}

// one element -> canonical 64-bit image (signed ints sign-extended, unsigned zero-extended,
// float widened to double)
__device__ __forceinline__ uint64_t load_elem(const DevCol& c, int64_t row) {
    uint64_t v;
    switch (c.stype) {
        case ST_I32: v = (uint64_t)(int64_t)__ldg((const int32_t*)c.values + row); break;
        case ST_U32: v = (uint64_t)__ldg((const uint32_t*)c.values + row); break;
        case ST_F32: v = f64_bits((double)__ldg((const float*)c.values + row)); break;
        case ST_U8: v = (uint64_t)__ldg((const uint8_t*)c.values + row); break;
        default: v = __ldg((const unsigned long long*)c.values + row); break;
    }
    return narrow_prim(v, c.prim);
}
__device__ __forceinline__ bool elem_is_null(const DevCol& c, int64_t row) {
    return c.validity != nullptr && !((__ldg(c.validity + (row >> 3)) >> (row & 7)) & 1);
}

// eight consecutive rows [8q, 8q+8) -> canonical images; nullmask bit j set = row j is NULL.
// Requires 32-byte aligned column buffers (checked by the host; otherwise the scalar path runs).
__device__ __forceinline__ void load_oct(const DevCol& c, int64_t q, uint64_t (&v)[8], uint32_t& nullmask) {
    switch (c.stype) {
        case ST_I32: {
            U32x8 r = ldg256_u32((const uint8_t*)c.values + q * 32);
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = (uint64_t)(int64_t)(int32_t)r.v[j];
        } break;
        case ST_U32: {
            U32x8 r = ldg256_u32((const uint8_t*)c.values + q * 32);
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = (uint64_t)r.v[j];
        } break;
        case ST_F32: {
            U32x8 r = ldg256_u32((const uint8_t*)c.values + q * 32);
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = f64_bits((double)__uint_as_float(r.v[j]));
        } break;
        case ST_U8: {
            unsigned long long r = __ldg((const unsigned long long*)c.values + q);
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = (r >> (8 * j)) & 0xFF;
        } break;
        default: {
            U64x4 a = ldg256_u64((const uint8_t*)c.values + q * 64);
            U64x4 b = ldg256_u64((const uint8_t*)c.values + q * 64 + 32);
#pragma unroll
            for (int j = 0; j < 4; j++) { v[j] = a.v[j]; v[4 + j] = b.v[j]; }
        } break;
    }
    if (c.prim == BK_INT8 || c.prim == BK_INT16 || c.prim == BK_UINT8 || c.prim == BK_UINT16 || c.prim == BK_BOOL) {
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = narrow_prim(v[j], c.prim);
    }
    nullmask = c.validity ? (uint32_t)(~__ldg(c.validity + q)) & 0xFFu : 0u;
}

// ------------------------------------------------------------------------------------------
// ExprValue arithmetic on canonical images
// ------------------------------------------------------------------------------------------
// comparison operators, src/expr/operators.cpp:84-100 (IEEE semantics for DOUBLE: NaN fails every
// ordered compare, != is true)
__device__ __forceinline__ bool cmp_vals(int op, int vclass, uint64_t a, uint64_t b) {
    if (vclass == VC_F64) {
        double x = bits_f64(a), y = bits_f64(b);
        switch (op) {
            case BK_FT_EQ: return x == y; case BK_FT_NE: return x != y;
            case BK_FT_GT: return x > y;  case BK_FT_GE: return x >= y;
            case BK_FT_LT: return x < y;  default: return x <= y;
        }
    }
    if (vclass == VC_U64) {
        switch (op) {
            case BK_FT_EQ: return a == b; case BK_FT_NE: return a != b;
            case BK_FT_GT: return a > b;  case BK_FT_GE: return a >= b;
            case BK_FT_LT: return a < b;  default: return a <= b;
        }
    }
    int64_t x = (int64_t)a, y = (int64_t)b;
    switch (op) {
        case BK_FT_EQ: return x == y; case BK_FT_NE: return x != y;
        case BK_FT_GT: return x > y;  case BK_FT_GE: return x >= y;
        case BK_FT_LT: return x < y;  default: return x <= y;
    }
}

__device__ __forceinline__ int prim_class(int prim) {
    switch (prim) {
        case BK_FLOAT: case BK_DOUBLE: return VC_F64;
        case BK_BOOL: case BK_UINT8: case BK_UINT16: case BK_UINT32: case BK_UINT64:
        case BK_TIMESTAMP: case BK_DATE: case BK_DATETIME: return VC_U64;
        default: return VC_I64;
    }
}
// double -> integer with the x86 semantics the reference build has (cvttsd2si: out-of-range and
// NaN give the "integer indefinite" value 0x8000...); C++ leaves those cases undefined.
__device__ __forceinline__ int64_t f64_to_i64_x86(double d) {
    if (!(d >= -9223372036854775808.0 && d < 9223372036854775808.0)) return (int64_t)0x8000000000000000ull;
    return (int64_t)d;
}
__device__ __forceinline__ uint64_t f64_to_u64_x86(double d) {
    // gcc: values >= 2^63 go through (int64)(d - 2^63) ^ 2^63; negatives wrap through the signed path
    if (d >= 9223372036854775808.0) return (uint64_t)f64_to_i64_x86(d - 9223372036854775808.0) ^ 0x8000000000000000ull;
    return (uint64_t)f64_to_i64_x86(d);
}
// ExprValue::cast_to (include/common/expr_value.h:502-611) for the numeric types
__device__ __forceinline__ uint64_t cast_prim(uint64_t v, int from, int to) {
    if (from != to && dt_is_family(from) && dt_is_family(to)) return dt_family_cast(v, from, to);   // DATE <-> DATETIME <-> TIMESTAMP (-> TIME)
    int fc = prim_class(from);
    if (to == BK_DOUBLE || to == BK_FLOAT) {
        double d = fc == VC_F64 ? bits_f64(v) : (fc == VC_U64 ? (double)v : (double)(int64_t)v);
        if (to == BK_FLOAT) d = (double)(float)d;
        return f64_bits(d);
    }
    if (to == BK_BOOL) return fc == VC_F64 ? (bits_f64(v) != 0.0) : (v != 0);
    uint64_t i;
    if (fc == VC_F64) {
        double d = bits_f64(v);
        if (to == BK_UINT64 || to == BK_DATETIME) i = f64_to_u64_x86(d);
        else if (to == BK_INT64) i = (uint64_t)f64_to_i64_x86(d);
        else { /* narrower targets convert through int32 / int64 on x86-64 */
            int64_t t = f64_to_i64_x86(d);
            if (to == BK_UINT32 || to == BK_TIMESTAMP || to == BK_DATE) i = (uint64_t)t;
            else i = (d >= -2147483648.0 && d < 2147483648.0) ? (uint64_t)(int64_t)(int32_t)d : 0xFFFFFFFF80000000ull;
        }
    } else i = v;
    switch (to) {
        case BK_INT8: return (uint64_t)(int64_t)(int8_t)i;
        case BK_INT16: return (uint64_t)(int64_t)(int16_t)i;
        case BK_INT32: case BK_TIME: return (uint64_t)(int64_t)(int32_t)i;
        case BK_UINT8: return (uint64_t)(uint8_t)i;
        case BK_UINT16: return (uint64_t)(uint16_t)i;
        case BK_UINT32: case BK_TIMESTAMP: case BK_DATE: return (uint64_t)(uint32_t)i;
        default: return i;
    }
}

// ------------------------------------------------------------------------------------------
// group table: open addressing, linear probing, per-slot state word (0 empty / 1 busy / 2 full).
// The same code serves the per-CTA shared-memory table and the global table.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t hash_key(const uint64_t* key, int kw) {
    uint64_t h = 0x9E3779B97F4A7C15ull;
#pragma unroll 1
    for (int i = 0; i < kw; i++) { h ^= key[i]; h *= 0xD6E8FEB86659FD93ull; h ^= h >> 32; }
    return (uint32_t)(h ^ (h >> 29));
}
__device__ __forceinline__ uint32_t hash_key1(uint64_t k) {
    uint64_t h = (k ^ 0x9E3779B97F4A7C15ull) * 0xD6E8FEB86659FD93ull;
    h ^= h >> 32;
    return (uint32_t)(h ^ (h >> 29));
}

template <bool SHARED>
struct TableMem {
    static __device__ __forceinline__ uint32_t ld_state(const uint32_t* p) {
        uint32_t v;
        if (SHARED) v = *(const volatile uint32_t*)p;
        else asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
        return v;
    }
    static __device__ __forceinline__ void publish(uint32_t* p) {
        if (SHARED) { __threadfence_block(); *(volatile uint32_t*)p = 2u; }
        else asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(2u) : "memory");
    }
    static __device__ __forceinline__ uint64_t ld_key(const uint64_t* p) {
        if (SHARED) return *(const volatile uint64_t*)p;
        return *(const volatile uint64_t*)p;
    }
};

// returns the slot of `key`, inserting it when absent; -1 when `max_probe` slots were examined
// without success (shared table: the row is routed to the global table; global table: overflow).
template <bool SHARED, int KW_STATIC>
__device__ __forceinline__ int table_upsert(uint32_t* state, uint64_t* keys, uint32_t cap_mask, const uint64_t* key,
                                            int kw_dyn, uint32_t h, int max_probe, uint32_t* n_groups) {
    const int kw = KW_STATIC > 0 ? KW_STATIC : kw_dyn;
    const uint32_t cap = cap_mask + 1;
    uint32_t slot = h & cap_mask;
    int probes = 0;
    while (probes < max_probe) {
        uint32_t s = TableMem<SHARED>::ld_state(state + slot);
        if (s == 0u) {
            uint32_t old = atomicCAS(state + slot, 0u, 1u);
            if (old == 0u) {
                for (int i = 0; i < kw; i++) keys[(size_t)i * cap + slot] = key[i];
                TableMem<SHARED>::publish(state + slot);
                if (n_groups) n_groups[GT_OCC_OFF + atomicAdd(n_groups, 1u)] = slot;   // (global table only: the occupied list)
                return (int)slot;
            }
            s = old;
        }
        if (s == 1u) continue;  // another thread is publishing this slot: re-read it
        bool same = true;
        for (int i = 0; i < kw; i++) same = same && (TableMem<SHARED>::ld_key(keys + (size_t)i * cap + slot) == key[i]);
        if (same) return (int)slot;
        slot = (slot + 1) & cap_mask;
        probes++;
    }
    return -1;
}

// ------------------------------------------------------------------------------------------
// accumulator lanes
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t lane_identity(int op) {
    switch (op) {   // (LN_HLL: 0 = no sketch)
        case LN_MIN_I64: return 0x7FFFFFFFFFFFFFFFull;
        case LN_MAX_I64: return 0x8000000000000000ull;
        case LN_MIN_U64: return 0xFFFFFFFFFFFFFFFFull;
        case LN_MAX_U64: return 0ull;
        case LN_MIN_F64: return 0x7FF0000000000000ull;  // +inf
        case LN_MAX_F64: return 0xFFF0000000000000ull;  // -inf
        // -0.0: the only double x with -0.0 + x == x for every x.  The reference's SUM takes its first value and adds the rest, so a SUM
        // over only -0.0 is -0.0; a +0.0 start would make it +0.0 (AVG starts from +0.0: extract_group normalises its sum)
        case LN_ADD_F64: return 0x8000000000000000ull;
        default: return 0ull;
    }
}
// thread-private combine (registers): r = r (op) v
__device__ __forceinline__ uint64_t lane_combine(int op, uint64_t r, uint64_t v) {
    switch (op) {
        case LN_ADD_I64: return r + v;
        case LN_ADD_F64: return f64_bits(bits_f64(r) + bits_f64(v));
        case LN_MIN_I64: return (int64_t)v < (int64_t)r ? v : r;
        case LN_MAX_I64: return (int64_t)v > (int64_t)r ? v : r;
        case LN_MIN_U64: return v < r ? v : r;
        case LN_MAX_U64: return v > r ? v : r;
        case LN_MIN_F64: return bits_f64(v) < bits_f64(r) ? v : r;   // ExprValue::compare: NaN never wins
        default: return bits_f64(v) > bits_f64(r) ? v : r;
    }
}
// 64-bit integer add in shared memory from two native 32-bit atomics (ATOMS.ADD) instead of the
// ATOMS.CAST.SPIN loop a 64-bit shared atomicAdd compiles to on sm_90a.
__device__ __forceinline__ void smem_add_u64(uint64_t* p, uint64_t v) {
    uint32_t* w = (uint32_t*)p;
    uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
    uint32_t old = atomicAdd(w, lo);
    uint32_t carry = (old + lo) < old ? 1u : 0u;
    if (hi + carry) atomicAdd(w + 1, hi + carry);
}
template <bool SHARED>
__device__ __forceinline__ void lane_atomic(int op, uint64_t* p, uint64_t v) {
    switch (op) {
        case LN_ADD_I64:
            if (SHARED) smem_add_u64(p, v); else atomicAdd((unsigned long long*)p, (unsigned long long)v);
            break;
        case LN_ADD_F64: atomicAdd((double*)p, bits_f64(v)); break;
        case LN_MIN_I64: atomicMin((long long*)p, (long long)v); break;
        case LN_MAX_I64: atomicMax((long long*)p, (long long)v); break;
        case LN_MIN_U64: atomicMin((unsigned long long*)p, (unsigned long long)v); break;
        case LN_MAX_U64: atomicMax((unsigned long long*)p, (unsigned long long)v); break;
        default: {  // f64 min / max: CAS loop with ExprValue::compare semantics
            unsigned long long* q = (unsigned long long*)p;
            unsigned long long cur = *(volatile unsigned long long*)q;
            for (;;) {
                bool better = op == LN_MIN_F64 ? bits_f64(v) < bits_f64(cur) : bits_f64(v) > bits_f64(cur);
                if (!better) break;
                unsigned long long prev = atomicCAS(q, cur, (unsigned long long)v);
                if (prev == cur) break;
                cur = prev;
            }
        } break;
    }
}

// convert an aggregate argument from the class it was evaluated in to the class of its lane
__device__ __forceinline__ uint64_t to_lane_class(uint64_t v, int from_class, int lane_class) {
    if (from_class == lane_class) return v;
    if (lane_class == VC_F64) return f64_bits(from_class == VC_U64 ? (double)v : (double)(int64_t)v);
    if (from_class == VC_F64) return lane_class == VC_U64 ? f64_to_u64_x86(bits_f64(v)) : (uint64_t)f64_to_i64_x86(bits_f64(v));
    return v;  // I64 <-> U64: same image
}

}  // namespace bk

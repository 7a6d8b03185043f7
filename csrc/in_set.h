// in_set.h — the hashed set an IN list is lowered to when it does not fit the program's constant pool (OP_IN_SET).  The host
// builds it once per IN expression when the plan is compiled (plan.cpp), bkgpu_open uploads it, and the interpreter probes it
// (interp.cuh); tests/cpp/in_set_check.cpp runs the same lookup on the host against a linear scan.
//
// Device image, 64-bit words:
//   [0]            log2 of the capacity (>= 1); the capacity is a power of two at least twice the number of distinct entries
//   [1]            1 when IN_SET_EMPTY itself is a member (it never occupies a slot)
//   [2, 2 + cap)   open-addressed slots of the entries' canonical images, IN_SET_EMPTY = free; multiplicative hash, linear probing
// Canonical images are the value class's (VClass): INT64 / UINT64 compare bit for bit, as OP_IN's cmp_vals does.  DOUBLE compares
// with ==, so -0.0 is stored and probed as 0.0, and NaN (equal to nothing) is dropped at build and misses as a probe.
#pragma once
#include <stdint.h>
#include <algorithm>
#include <vector>
#include "dev_types.h"

#if defined(__CUDACC__)
#define BK_HD __host__ __device__ __forceinline__
#else
#define BK_HD inline
#endif

namespace bk {

constexpr int IN_SET_HEADER = 2;                          // words before the slots
constexpr uint64_t IN_SET_EMPTY = 0x7FF8A5A5A5A5A5A5ull;  // a NaN image: never a DOUBLE member, and an unlikely integer
constexpr uint64_t IN_SET_MUL = 0x9E3779B97F4A7C15ull;    // 2^64 / golden ratio

BK_HD bool in_set_is_nan(uint64_t x, int vclass) { return vclass == VC_F64 && (x & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull; }
BK_HD uint64_t in_set_canon(uint64_t x, int vclass) { return vclass == VC_F64 && x == 0x8000000000000000ull ? 0 : x; }
BK_HD uint64_t in_set_home(uint64_t x, int log2) { return (x * IN_SET_MUL) >> (64 - log2); }

BK_HD bool in_set_contains(const uint64_t* set, uint64_t x, int vclass) {
    if (in_set_is_nan(x, vclass)) return false;
    x = in_set_canon(x, vclass);
#if defined(__CUDA_ARCH__)
    if (x == IN_SET_EMPTY) return __ldg((const unsigned long long*)set + 1) != 0;
    const int log2 = (int)__ldg((const unsigned long long*)set);
#else
    if (x == IN_SET_EMPTY) return set[1] != 0;
    const int log2 = (int)set[0];
#endif
    const uint64_t mask = ((uint64_t)1 << log2) - 1;
    const uint64_t* slots = set + IN_SET_HEADER;
    for (uint64_t i = in_set_home(x, log2);; i = (i + 1) & mask) {   // (at least half the slots are free: the walk ends)
#if defined(__CUDA_ARCH__)
        const uint64_t s = __ldg((const unsigned long long*)slots + i);
#else
        const uint64_t s = slots[i];
#endif
        if (s == x) return true;
        if (s == IN_SET_EMPTY) return false;
    }
}

// the device image of the set of `n` entries (canonical images of class `vclass`); duplicates collapse.  `n_distinct` receives the
// number of distinct members, the sentinel and excluding NaN.
inline std::vector<uint64_t> in_set_build(const uint64_t* v, size_t n, int vclass, uint32_t* n_distinct) {
    std::vector<uint64_t> keys;
    keys.reserve(n);
    for (size_t i = 0; i < n; i++) if (!in_set_is_nan(v[i], vclass)) keys.push_back(in_set_canon(v[i], vclass));
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    *n_distinct = (uint32_t)keys.size();
    int log2 = 1;
    while (((uint64_t)1 << log2) < 2 * (uint64_t)keys.size()) log2++;
    const uint64_t cap = (uint64_t)1 << log2, mask = cap - 1;
    std::vector<uint64_t> img(IN_SET_HEADER + cap, IN_SET_EMPTY);
    img[0] = (uint64_t)log2;
    img[1] = 0;
    uint64_t* slots = img.data() + IN_SET_HEADER;
    for (uint64_t k : keys) {
        if (k == IN_SET_EMPTY) { img[1] = 1; continue; }
        uint64_t i = in_set_home(k, log2);
        while (slots[i] != IN_SET_EMPTY) i = (i + 1) & mask;
        slots[i] = k;
    }
    return img;
}

}  // namespace bk

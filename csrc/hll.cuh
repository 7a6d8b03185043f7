// hll.cuh — hll_add_agg's per-row work, shared by the host and the device: the value hash (ExprValue::hash, the reference's
// include/common/expr_value.h:667-702: MurmurHash3_x64_128 of the value's native bytes, seed 0x110, first half) and the register
// it feeds (hll_pat_len, src/common/hll_common.cpp:41-56).  Only keys of at most 8 bytes arrive here, so the hash has no 16-byte
// block loop: the key is the algorithm's tail.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define BK_HD __host__ __device__ __forceinline__
#else
#define BK_HD inline
#endif

namespace bk {

constexpr int HLL_P = 14;                               // register index bits
constexpr int HLL_REGISTERS = 1 << HLL_P;               // 16384 one-byte registers per sketch
constexpr int HLL_HDR_BYTES = 16;                       // "HYLL", encoding, 3 unused bytes, 8 bytes of cached cardinality
constexpr int HLL_RAW_BYTES = HLL_HDR_BYTES + HLL_REGISTERS;   // 16400: the RAW sketch hll_row_init builds
constexpr uint8_t HLL_ENC_RAW = 255;
constexpr uint32_t HLL_SEED = 0x110;

BK_HD uint64_t hll_rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
BK_HD uint64_t hll_fmix64(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return k;
}

// MurmurHash3_x64_128(key, len, seed)[0] for 1 <= len <= 8, the key being the low `len` bytes of `v` (little-endian)
BK_HD uint64_t hll_hash(uint64_t v, int len, uint32_t seed = HLL_SEED) {
    uint64_t h1 = seed, h2 = seed;
    uint64_t k1 = len >= 8 ? v : (v & ((1ull << (8 * len)) - 1ull));
    k1 *= 0x87c37b91114253d5ull; k1 = hll_rotl64(k1, 31); k1 *= 0x4cf5ad432745937full;
    h1 ^= k1;
    h1 ^= (uint64_t)len; h2 ^= (uint64_t)len;
    h1 += h2; h2 += h1;
    h1 = hll_fmix64(h1); h2 = hll_fmix64(h2);
    h1 += h2;
    return h1;
}

// the register a hash feeds and the value it offers: 1 + trailing zeros of the bits above the index, capped at 51 by a guard bit
BK_HD int hll_pat_len(uint64_t h, uint32_t* reg) {
    *reg = (uint32_t)(h & (HLL_REGISTERS - 1));
    const uint64_t x = (h >> HLL_P) | (1ull << (64 - HLL_P));
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)x);
#else
    return __builtin_ctzll(x) + 1;
#endif
}

// bytes of the value the reference hashes, by the argument's type after inference (ExprValue::hash's switch); 0 = not hashed here
BK_HD int hll_key_bytes(int prim) {
    switch (prim) {
        case 2 /*BOOL*/: case 3 /*INT8*/: case 7 /*UINT8*/: return 1;
        case 4 /*INT16*/: case 8 /*UINT16*/: return 2;
        case 5 /*INT32*/: case 9 /*UINT32*/: case 11 /*FLOAT*/: case 15 /*TIMESTAMP*/: case 16 /*DATE*/: case 18 /*TIME*/: return 4;
        case 6 /*INT64*/: case 10 /*UINT64*/: case 12 /*DOUBLE*/: case 14 /*DATETIME*/: return 8;
        default: return 0;
    }
}

}  // namespace bk

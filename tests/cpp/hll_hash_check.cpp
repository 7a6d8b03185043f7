// A second restatement of MurmurHash3_x64_128 (any key length, byte-wise, in plain C), checked against SMHasher's published
// verification value and used to pin csrc/hll.cuh's host copy of hll_add_agg's hash and register choice.
//   g++ -std=c++17 -I csrc tests/cpp/hll_hash_check.cpp -o hll_hash_check && ./hll_hash_check
// Prints "verification 0x........", then one line per vector: "width value hash index count"; exits 1 on a mismatch.
#include <inttypes.h>
#include <stdio.h>
#include <string.h>
#include "hll.cuh"

static uint64_t rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
static uint64_t fmix(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
    return k;
}
static uint64_t le64(const unsigned char* p, int n) {   // n <= 8 bytes, little-endian
    uint64_t v = 0;
    for (int i = n - 1; i >= 0; i--) v = (v << 8) | p[i];
    return v;
}
static void murmur3_x64_128(const void* key, int len, uint32_t seed, uint64_t out[2]) {
    const unsigned char* d = (const unsigned char*)key;
    const uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
    uint64_t h1 = seed, h2 = seed;
    const int nb = len / 16;
    for (int i = 0; i < nb; i++) {
        uint64_t k1 = le64(d + 16 * i, 8), k2 = le64(d + 16 * i + 8, 8);
        k1 *= c1; k1 = rotl(k1, 31); k1 *= c2; h1 ^= k1;
        h1 = rotl(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
        k2 *= c2; k2 = rotl(k2, 33); k2 *= c1; h2 ^= k2;
        h2 = rotl(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
    }
    const unsigned char* t = d + 16 * nb;
    const int rest = len & 15;
    if (rest > 8) { uint64_t k2 = le64(t + 8, rest - 8); k2 *= c2; k2 = rotl(k2, 33); k2 *= c1; h2 ^= k2; }
    if (rest > 0) { uint64_t k1 = le64(t, rest > 8 ? 8 : rest); k1 *= c1; k1 = rotl(k1, 31); k1 *= c2; h1 ^= k1; }
    h1 ^= (uint64_t)len; h2 ^= (uint64_t)len;
    h1 += h2; h2 += h1;
    h1 = fmix(h1); h2 = fmix(h2);
    h1 += h2; h2 += h1;
    out[0] = h1; out[1] = h2;
}

int main() {
    unsigned char key[256], hashes[256 * 16];
    for (int i = 0; i < 256; i++) {
        key[i] = (unsigned char)i;
        uint64_t o[2];
        murmur3_x64_128(key, i, 256 - i, o);
        memcpy(hashes + 16 * i, o, 16);
    }
    uint64_t fin[2];
    murmur3_x64_128(hashes, 256 * 16, 0, fin);
    const uint32_t verification = (uint32_t)fin[0];
    printf("verification 0x%08" PRIX32 "\n", verification);
    int bad = verification != 0x6384BA69u;
    const uint64_t values[] = {0, 1, 2, 0x7F, 0x80, 0xFF, 0x1234, 0xFFFF, 0x7FFFFFFF, 0x80000000ULL, 0xFFFFFFFFULL, 0x3FF0000000000000ULL /* 1.0 */,
                               0x8000000000000000ULL /* -0.0, INT64_MIN */, 0x7FFFFFFFFFFFFFFFULL, 0xFFFFFFFFFFFFFFFFULL, 0x7FF8000000000000ULL /* NaN */,
                               0x7FC00000ULL /* float NaN */, 0x0123456789ABCDEFULL, 20241231ULL};
    const int widths[] = {1, 2, 4, 8};
    for (int w : widths)
        for (uint64_t v : values) {
            unsigned char b[8];
            memcpy(b, &v, 8);   // (little-endian host: the value's low bytes)
            uint64_t o[2];
            murmur3_x64_128(b, w, bk::HLL_SEED, o);
            uint32_t idx = 0;
            const int count = bk::hll_pat_len(o[0], &idx);
            int tz = 0;
            while (tz < 50 && !(((o[0] >> 14) >> tz) & 1)) tz++;
            if (bk::hll_hash(v, w) != o[0] || idx != (uint32_t)(o[0] & 0x3FFF) || count != tz + 1) { bad = 1; printf("MISMATCH "); }
            printf("%d 0x%016" PRIx64 " 0x%016" PRIx64 " %u %d\n", w, v, o[0], idx, count);
        }
    return bad;
}

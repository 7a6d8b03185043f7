// sort_key_check.cpp — csrc/sort_key.h's key image against ExprValue::compare (`a > b ? 1 : a < b ? -1 : 0`, what MemRowCompare asks of
// every ORDER BY key), for every value class and both directions: all pairs of a list of special values and 10^5 seeded random pairs must
// satisfy  sign(image(a) - image(b)) == sign(asc ? cmp(a, b) : -cmp(a, b)).  NaN is left out of that property (the reference's compare is
// not an order there) and pinned separately: a NaN's image depends on its bits only, and every NaN sorts outside [-Inf, +Inf].
// Prints "sort_key_check ok" and the case count.
#include <stdio.h>
#include <string.h>
#include <cfloat>
#include <limits>
#include <random>
#include <vector>
#include "sort_key.h"

using namespace bk;

static uint64_t dbits(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
static double bitsd(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }
static bool is_nan_bits(uint64_t u) { return (u & 0x7FFFFFFFFFFFFFFFull) > 0x7FF0000000000000ull; }

static long n_cases = 0, n_fail = 0;

template <class V> static int cmp3(V a, V b) { return a > b ? 1 : (a < b ? -1 : 0); }   // ExprValue::compare
static int cmp_class(uint64_t a, uint64_t b, int vc) {
    if (vc == VC_I64) return cmp3((int64_t)a, (int64_t)b);
    if (vc == VC_U64) return cmp3(a, b);
    return cmp3(bitsd(a), bitsd(b));
}

static void check_pair(uint64_t a, uint64_t b, int vc) {
    for (int desc = 0; desc < 2; desc++) {
        n_cases++;
        const int want = desc ? -cmp_class(a, b, vc) : cmp_class(a, b, vc);
        const int got = cmp3(key_image(a, vc, desc), key_image(b, vc, desc));
        if (want != got && n_fail++ < 20)
            printf("FAIL class=%d desc=%d a=0x%016llx b=0x%016llx want=%d got=%d\n", vc, desc, (unsigned long long)a, (unsigned long long)b, want, got);
    }
}

int main() {
    std::mt19937_64 rng(20261016);
    const uint64_t i64_min = 0x8000000000000000ull, i64_max = 0x7FFFFFFFFFFFFFFFull, u64_max = ~0ull;
    const std::vector<uint64_t> int_special = {0, 1, u64_max /* -1 */, 2, u64_max - 1, i64_min, i64_max, i64_min + 1, i64_max - 1, 255, 256, 1ull << 32, (1ull << 32) - 1};
    const double dmin = std::numeric_limits<double>::denorm_min(), inf = std::numeric_limits<double>::infinity();
    const std::vector<uint64_t> dbl_special = {dbits(0.0), dbits(-0.0), dbits(1.0), dbits(-1.0), dbits(dmin), dbits(-dmin), dbits(DBL_MIN), dbits(-DBL_MIN),
                                               dbits(DBL_MAX), dbits(-DBL_MAX), dbits(inf), dbits(-inf), dbits(0.5), dbits(-0.5), dbits(1e-300), dbits(-1e300)};
    for (int vc : {VC_I64, VC_U64, VC_F64}) {
        const std::vector<uint64_t>& special = vc == VC_F64 ? dbl_special : int_special;
        for (uint64_t a : special) for (uint64_t b : special) check_pair(a, b, vc);
        auto rand_value = [&]() -> uint64_t {
            const uint64_t r = rng();
            if (r % 8 == 0) return special[rng() % special.size()];
            if (r % 8 <= 3) {   // any bit pattern (doubles: every binade, denormals; no NaN)
                uint64_t x = rng();
                while (vc == VC_F64 && is_nan_bits(x)) x = rng();
                return x;
            }
            const int64_t small = (int64_t)(rng() % 2001) - 1000;   // near ties
            return vc == VC_F64 ? dbits((double)small / 8.0) : (uint64_t)small;
        };
        for (int i = 0; i < 100000; i++) check_pair(rand_value(), rand_value(), vc);
    }
    // NaN: the image is a function of the bits only (equal bits, equal images; different bits, different images), negative NaNs sort
    // below -Inf and positive NaNs above +Inf ascending, mirrored descending
    const std::vector<uint64_t> nans = {dbits(std::numeric_limits<double>::quiet_NaN()), 0x7FF0000000000001ull, 0x7FFFFFFFFFFFFFFFull, 0xFFF8000000000000ull,
                                        0xFFF0000000000001ull, 0xFFFFFFFFFFFFFFFFull};
    for (int desc = 0; desc < 2; desc++) {
        const uint64_t lo = key_image(dbits(desc ? inf : -inf), VC_F64, desc), hi = key_image(dbits(desc ? -inf : inf), VC_F64, desc);
        for (uint64_t a : nans) {
            n_cases++;
            const uint64_t ia = key_image(a, VC_F64, desc);
            const bool below = ((a >> 63) != 0) != (desc != 0);   // ascending: the negative ones
            if (!(below ? ia < lo : ia > hi) && n_fail++ < 20) printf("FAIL NaN 0x%016llx desc=%d sorts inside [-Inf, +Inf]\n", (unsigned long long)a, desc);
            for (uint64_t b : nans) {
                n_cases++;
                if ((ia == key_image(b, VC_F64, desc)) != (a == b) && n_fail++ < 20)
                    printf("FAIL NaN images 0x%016llx 0x%016llx desc=%d\n", (unsigned long long)a, (unsigned long long)b, desc);
            }
        }
    }
    if (n_fail) { printf("sort_key_check: %ld of %ld cases failed\n", n_fail, n_cases); return 1; }
    printf("sort_key_check ok %ld cases\n", n_cases);
    return 0;
}

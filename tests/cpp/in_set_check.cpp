// in_set_check.cpp — csrc/in_set.h's lookup and OP_IN's three-valued result over it, against a linear scan with OP_IN's comparison
// (cmp_vals: bit equality for INT64 / UINT64 images, == for DOUBLE), for every value class.  Prints "in_set_check ok" and the case count.
#include <stdio.h>
#include <string.h>
#include <limits>
#include <random>
#include <vector>
#include "in_set.h"

using namespace bk;

static uint64_t dbits(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
static double bitsd(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }

static long n_cases = 0, n_fail = 0;

// OP_IN's answer: 1 = TRUE, 0 = FALSE, -1 = NULL (a NULL probe, or a miss when the list held a NULL)
static int three_valued(bool probe_null, bool found, bool has_null) { return probe_null ? -1 : (found ? 1 : (has_null ? -1 : 0)); }

static void check_list(const char* what, const std::vector<uint64_t>& list, std::vector<uint64_t> probes, int vc) {
    uint32_t distinct = 0;
    const std::vector<uint64_t> img = in_set_build(list.data(), list.size(), vc, &distinct);
    const uint64_t cap = img.size() - IN_SET_HEADER;
    std::vector<uint64_t> members;   // distinct canonical non-NaN entries
    for (uint64_t v : list) if (!in_set_is_nan(v, vc)) members.push_back(in_set_canon(v, vc));
    std::sort(members.begin(), members.end());
    members.erase(std::unique(members.begin(), members.end()), members.end());
    if (distinct != members.size() || (cap & (cap - 1)) != 0 || cap < 2 * (uint64_t)distinct || cap != ((uint64_t)1 << img[0])) {
        printf("FAIL %s: layout distinct=%u members=%zu cap=%llu\n", what, distinct, members.size(), (unsigned long long)cap);
        n_fail++;
    }
    // probes: members, their neighbours, and what the caller adds
    const size_t step = list.size() > 200 ? list.size() / 200 : 1;
    for (size_t i = 0; i < list.size(); i += step) { probes.push_back(list[i]); probes.push_back(list[i] + 1); probes.push_back(list[i] - 1); }
    for (uint64_t x : probes) {
        bool lin = false;   // the linear scan, with OP_IN's comparison
        for (uint64_t v : list) if (vc == VC_F64 ? bitsd(v) == bitsd(x) : v == x) { lin = true; break; }
        const bool got = in_set_contains(img.data(), x, vc);
        for (int has_null = 0; has_null < 2; has_null++)
            for (int pn = 0; pn < 2; pn++) {
                n_cases++;
                const int w = three_valued(pn, lin, has_null), g = three_valued(pn, got, has_null);
                if (w != g && n_fail++ < 20)
                    printf("FAIL %s: class=%d n=%zu null=%d probe=0x%llx probe_null=%d want=%d got=%d\n", what, vc, list.size(), has_null,
                           (unsigned long long)x, pn, w, g);
            }
    }
}

int main() {
    std::mt19937_64 rng(20261016);
    const uint64_t i64_min = 0x8000000000000000ull, i64_max = 0x7FFFFFFFFFFFFFFFull, u64_max = ~0ull;
    std::vector<uint64_t> int_special = {0, 1, u64_max, i64_min, i64_max, i64_min + 1, i64_max - 1, IN_SET_EMPTY, IN_SET_EMPTY + 1, IN_SET_EMPTY - 1};
    const double dmin = std::numeric_limits<double>::denorm_min(), inf = std::numeric_limits<double>::infinity();
    std::vector<uint64_t> dbl_special = {dbits(0.0), dbits(-0.0), dbits(inf), dbits(-inf), dbits(dmin), dbits(-dmin), dbits(2.2250738585072009e-308),
                                         dbits(std::numeric_limits<double>::quiet_NaN()), 0x7FF0000000000001ull, 0xFFF8000000000000ull, IN_SET_EMPTY,
                                         dbits(1.0), dbits(-1.0), dbits(std::numeric_limits<double>::max()), dbits(-std::numeric_limits<double>::max())};
    const size_t sizes[] = {1, 2, 3, 7, 64, 65, 255, 256, 1000, 4096, 65537, 1000000};
    for (int vc : {VC_I64, VC_U64, VC_F64}) {
        const std::vector<uint64_t>& special = vc == VC_F64 ? dbl_special : int_special;
        auto rand_value = [&]() -> uint64_t {
            if (vc != VC_F64) return rng() % 4 == 0 ? rng() : (uint64_t)(int64_t)((int64_t)(rng() % 2000001) - 1000000);
            const uint64_t r = rng();
            if (r % 8 == 0) return special[rng() % special.size()];
            if (r % 8 == 1) return rng();   // any bit pattern: NaNs and denormals included
            return dbits((double)((int64_t)(rng() % 2000001) - 1000000) / 4.0);
        };
        for (size_t n : sizes) {
            std::vector<uint64_t> probes = special;
            for (int i = 0; i < 200; i++) probes.push_back(rand_value());
            // distinct-ish random values with the special ones mixed in
            std::vector<uint64_t> list;
            for (size_t i = 0; i < n; i++) list.push_back(i < special.size() && n >= 64 ? special[i] : rand_value());
            check_list("random", list, probes, vc);
            // heavy duplicates: values drawn from a handful
            std::vector<uint64_t> few;
            for (int i = 0; i < 5; i++) few.push_back(rand_value());
            for (size_t i = 0; i < n; i++) list[i] = few[rng() % few.size()];
            check_list("duplicates", list, probes, vc);
            // every entry equal
            for (size_t i = 0; i < n; i++) list[i] = few[0];
            check_list("all equal", list, probes, vc);
        }
        // the sentinel alone, and each special value alone, as a member and as a probe
        for (uint64_t s : special) check_list("special alone", std::vector<uint64_t>(3, s), special, vc);
        check_list("specials", special, special, vc);
    }
    if (n_fail) { printf("in_set_check: %ld of %ld cases failed\n", n_fail, n_cases); return 1; }
    printf("in_set_check ok %ld cases\n", n_cases);
    return 0;
}

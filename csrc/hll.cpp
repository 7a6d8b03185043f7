// hll.cpp — bkgpu_hll_estimate: the reference's hll_estimate (src/common/hll_common.cpp:523-600, Redis's histogram estimator) over a
// RAW sketch as hll_add_agg returns it.  Host code: an adapter or the benchmark reads the cardinality of a returned sketch.
#include <math.h>
#include <string.h>
#include "hll.cuh"
#include "../include/bkgpu.h"

namespace {

constexpr int HLL_Q = 64 - bk::HLL_P;   // hash bits left for the run of zeros: register values 0 .. HLL_Q + 1
constexpr double HLL_ALPHA_INF = 0.721347520444481703680;   // 0.5 / ln(2)

double hll_sigma(double x) {
    if (x == 1.) return INFINITY;
    double z_prev = 0.0, y = 1, z = x;
    do { x *= x; z_prev = z; z += x * y; y += y; } while (z_prev != z);
    return z;
}

double hll_tau(double x) {
    if (x == 0. || x == 1.) return 0.;
    double z_prev = 0.0, y = 1.0, z = 1 - x;
    do { x = sqrt(x); z_prev = z; y *= 0.5; z -= pow(1 - x, 2) * y; } while (z_prev != z);
    return z / 3;
}

}  // namespace

extern "C" int bkgpu_hll_estimate(const uint8_t* sketch, size_t len, uint64_t* estimate) {
    if (!sketch || !estimate || len != (size_t)bk::HLL_RAW_BYTES || memcmp(sketch, "HYLL", 4) != 0 || sketch[4] != bk::HLL_ENC_RAW) return BKGPU_EINVAL;
    uint64_t card = 0;
    if (!(sketch[15] & 0x80)) {   // the cached cardinality is valid
        for (int i = 0; i < 8; i++) card |= (uint64_t)sketch[8 + i] << (8 * i);
        *estimate = card;
        return BKGPU_OK;
    }
    const double m = bk::HLL_REGISTERS;
    int histo[64] = {0};
    for (int i = 0; i < bk::HLL_REGISTERS; i++) {
        const uint8_t r = sketch[bk::HLL_HDR_BYTES + i];
        if (r > HLL_Q + 1) return BKGPU_EINVAL;   // (no hash gives a register beyond 51)
        histo[r]++;
    }
    double z = m * hll_tau((m - histo[HLL_Q + 1]) / m);
    for (int j = HLL_Q; j >= 1; --j) { z += histo[j]; z *= 0.5; }
    z += m * hll_sigma(histo[0] / m);
    if (!(fabs(z) < 1e-9)) card = (uint64_t)llroundl(HLL_ALPHA_INF * m * m / z);   // (the reference's float_equal; an empty sketch gives z = inf, so 0)
    *estimate = card;
    return BKGPU_OK;
}

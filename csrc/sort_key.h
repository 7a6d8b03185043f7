// sort_key.h — the order-preserving 64-bit image of a sort key (ORDER BY / top-k, the multi-GPU k-row merge and the window stage's sort all
// compare these images as unsigned integers); tests/cpp/sort_key_check.cpp checks it on the host against ExprValue::compare.
//
// For two non-NaN values a, b of one value class:  image(a) < image(b)  <=>  MemRowCompare orders a before b (ascending; descending is the
// complement), and image(a) == image(b) <=> they compare equal.  -0.0 and +0.0 compare equal in the reference (`_u.double_val > other ? 1 :
// (< ? -1 : 0)`), so both map to +0.0's image: ties between them fall through to the next key / the arrival index.  Payload columns are
// gathered from the rows, not from images, so a returned -0.0 keeps its sign.  NaN has no place in the reference's order (compare says 0
// against everything); its image is the IEEE bit order's: negative NaNs below -Inf, positive NaNs above +Inf.
#pragma once
#include <stdint.h>
#include "dev_types.h"

#if defined(__CUDACC__)
#define BK_HD __host__ __device__ __forceinline__
#else
#define BK_HD inline
#endif

namespace bk {

BK_HD uint64_t key_image(uint64_t v, int vclass, int desc) {
    uint64_t t;
    if (vclass == VC_F64) {
        if ((v << 1) == 0) v = 0;   // -0.0 == +0.0
        t = (v >> 63) ? ~v : (v | 0x8000000000000000ull);
    } else if (vclass == VC_I64) t = v ^ 0x8000000000000000ull;
    else t = v;
    return desc ? ~t : t;
}

}  // namespace bk

// prims.cuh — device primitives of ORDER BY, the window stage and rb_build_agg (prims.cu): radix sort, prefix sum, row ids, null bitmaps
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "../include/bkgpu.h"

namespace bk {

// CTAs of 256 threads for a grid-stride loop over n items: at least one, at most `per_sm` per SM
int grid_for(int64_t n, int sm, int per_sm);

__global__ void k_iota(uint32_t* ids, int64_t n);   // ids[i] = i
// null BYTES (1 = NULL) -> Arrow validity bitmap (bit set = valid); *any_null = 1 when one is NULL (any_null may be nullptr)
__global__ void k_pack_null_bytes(const uint8_t* nb, int64_t n, uint8_t* bitmap, uint32_t* any_null);

// exclusive prefix sum of d[0, n) in place, for uint32_t and uint64_t; `sums` holds scan_scratch(n) entries
template <typename T> cudaError_t scan_excl(T* d, int64_t n, T* sums, int sm, cudaStream_t s);
int64_t scan_scratch(int64_t n);

// the radix sort keeps a tile's prefix count in a 30-bit field
constexpr int64_t RADIX_MAX_KEYS = ((int64_t)1 << 30) - 1;
// the radix sort's device scratch (the plan's buffers, grown as its sorts need): histograms and the look-back status
struct RadixScratch {
    void* hist = nullptr; size_t hist_cap = 0;
    void* status = nullptr; size_t status_cap = 0;
};
// Stable LSD radix sort of n <= RADIX_MAX_KEYS 64-bit keys in keys[cur], 8 bits per pass, keys[cur ^ 1] the second buffer; with ids
// (nullptr: keys alone), ids[cur] travel with their keys.  Runs on p->stream.  Returns the buffer that holds the result, or a BKGPU
// code < 0 (set by p->fail).  Counts its launches in stats->kernel_launches and, with `bytes`, the bytes its passes move in *bytes.
int radix_sort(bkgpu_plan* p, uint64_t* const keys[2], uint32_t* const ids[2], int cur, int64_t n, RadixScratch& scratch, bkgpu_stats* stats,
               int64_t* bytes);

}  // namespace bk

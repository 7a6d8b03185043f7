// prims.cuh — device primitives of ORDER BY, the window stage, the hash join and rb_build_agg (prims.cu): radix sort, prefix sum, row ids,
// and the row store with its null bitmaps
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <vector>
#include "../include/bkgpu.h"
#include "plan.h"

namespace bk {

// CTAs of 256 threads for a grid-stride loop over n items: at least one, at most `per_sm` per SM
int grid_for(int64_t n, int sm, int per_sm);

__global__ void k_iota(uint32_t* ids, int64_t n);   // ids[i] = i
// null BYTES (1 = NULL) -> Arrow validity bitmap (bit set = valid); *any_null = 1 when one is NULL (any_null may be nullptr)
__global__ void k_pack_null_bytes(const uint8_t* nb, int64_t n, uint8_t* bitmap, uint32_t* any_null);

// the payload gathers of ORDER BY / top-k / filter-only (sort.cu): rows of the batch columns `cols`, or of the rows kept from earlier
// batches, into value / null-byte columns
struct GatherArgs {
    DevCol cols[MAX_COLS]; int32_t n_cols; uint64_t row_base; int64_t nrows;
    uint8_t* dst_vals[MAX_COLS]; uint8_t* dst_null[MAX_COLS];
    const uint8_t* old_vals[MAX_COLS]; const uint8_t* old_null[MAX_COLS];
    const uint64_t* old_idx; uint32_t old_n;
};
// dst row dst_off + i = row sel[i] of every column of g
__global__ void k_gather_sel(GatherArgs g, const uint32_t* sel, uint64_t n, uint64_t dst_off);

// Rows on the device, in the one format the library keeps them in: per column its values and null BYTES (1 = NULL), and the Arrow
// validity bitmap packed from those bytes for the kernels that read DevCols.  Holds ORDER BY's / the window stage's retained rows
// (sort.cu), the hash join's build sides and gathered chunk (join.cu) and the post fragment's input (agg.cu, join.cu, window.cu).
// The buffers come from the plan's allocator, which returns them at bkgpu_close.
struct RowStore {
    struct Col {
        int prim = -1;                   // -1: a column the store does not hold (a join side holds its own table's columns only)
        uint8_t *vals = nullptr, *nulls = nullptr, *bitmap = nullptr;
        int64_t cap = 0, null_cap = 0;   // rows the values / the null bytes and bitmap have room for
        bool nullable = false;           // an appended batch came with a validity bitmap (store_append)
    };
    std::vector<Col> cols;
    int64_t rows = 0;                    // rows held (the chunk and the post input hold none: every use refills them)
    int64_t cap = 0;                     // rows every held column has room for (store_retain)
};
void store_init(RowStore& s, const std::vector<ColRef>& cols);
// room for `need` rows in column i, and in its null bytes and bitmap when `nulls`: a buffer with less room is reallocated with room for
// `cap` rows, the s.rows rows it holds copied over
int store_reserve(bkgpu_plan* p, RowStore& s, size_t i, int64_t need, int64_t cap, bool nulls);
// retention: room for `need` rows in every held column, the rows held kept; a store that must grow grows to max(need, 2 cap, 65536) rows
int store_retain(bkgpu_plan* p, RowStore& s, int64_t need);
// n rows of one bound batch column appended to column i at row s.rows (the caller advances s.rows): device input by a copy and the unpack
// kernel, host input by a copy of the values and of null bytes built on the host (counted in p->stats.h2d_bytes)
int store_append(bkgpu_plan* p, RowStore& s, size_t i, const bkgpu_column& in, int64_t n, bool on_device);
// column i's first n rows as a DevCol, the bitmap packed from their null bytes (CTAs: grid_for(…, p->sm_count, per_sm)); *any_null
// (device, may be nullptr) is set when one of them is NULL
int store_pack(bkgpu_plan* p, const RowStore& s, size_t i, int64_t n, int per_sm, uint32_t* any_null, DevCol* out);
// column i as a DevCol whose bitmap (packed by store_pack) is read only when an appended batch brought NULLs: a bitmap packed by an
// earlier run of the plan must not mask this run's rows
DevCol store_col(const RowStore& s, size_t i);
// dst_vals / dst_nulls [0, n) = the values / null bytes of rows perm[0, n) of column `src`
int store_gather(bkgpu_plan* p, const RowStore::Col& src, const uint32_t* perm, int64_t n, uint8_t* dst_vals, uint8_t* dst_nulls);
// rows [skip, skip + n) of the columns of `s` (through the device permutation `perm` when not nullptr) to the host as the plan's result
// (p->result, result_rows), column c described by desc[c] with kind 0
int store_copy_out(bkgpu_plan* p, const RowStore& s, const std::vector<ColRef>& desc, const uint32_t* perm, int64_t n, int64_t skip);

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

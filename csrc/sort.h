// sort.h — K5 (ORDER BY / top-k) and K1 (filter-only stream compaction): host entry points used by api.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "../include/bkgpu.h"
#include "plan.h"

namespace bk {

struct SortState;  // opaque (sort.cu)

struct SortOutCol {
    int tuple_id, slot_id, prim, elem;
    std::vector<uint8_t> values;
    std::vector<uint8_t> validity;  // LSB bitmap, empty = all valid
};

int  sort_open(const Compiled& c, int device, cudaStream_t stream, int64_t region_base, SortState** out, std::string& err);
int  sort_push(SortState* s, const DevCol* cols, int64_t nrows, cudaStream_t stream, bkgpu_stats* stats, std::string& err);
int  sort_finish(SortState* s, void* nccl_comm, int nranks, cudaStream_t stream, bkgpu_stats* stats,
                 std::vector<SortOutCol>& out, int64_t* nrows, std::string& err);
size_t sort_partial_bytes(SortState* s);
int  sort_partial_export(SortState* s, void* dev_dst, cudaStream_t stream, std::string& err);
int  sort_partial_merge(SortState* s, const void* dev_src, int nranks, cudaStream_t stream,
                        std::vector<SortOutCol>& out, int64_t* nrows, std::string& err);
int  sort_reset(SortState* s, cudaStream_t stream, std::string& err);

// ---- the window stage (window.cu) over a SortState's retained rows (a PK_WINDOW plan retains its filtered rows like a full sort) ----
// the retained rows as device columns with validity bitmaps; the bitmaps land in `scratch` (sort_free_scratch releases them)
int  sort_retained_cols(SortState* s, cudaStream_t stream, std::vector<DevCol>& cols, std::vector<void*>& scratch, int64_t* nrows, std::string& err);
// the retained columns' value buffers and null BYTES (1 = NULL), in arrival order
int  sort_retained_raw(SortState* s, std::vector<uint8_t*>& vals, std::vector<uint8_t*>& nulls);
void sort_free_scratch(SortState* s, std::vector<void*>& scratch);
// stable LSD radix sort of the row ids `ids` (device, n entries, the current order) by `keys`; key k's image is output keys[k].out_reg
// of program progs[k] over `cols`
int  sort_stable_ids(SortState* s, const DevCol* cols, int64_t n, const std::vector<SortKey>& keys, const std::vector<const Program*>& progs,
                     uint32_t* ids, cudaStream_t stream, bkgpu_stats* stats, std::string& err);
// rows perm[skip .. skip+n) of value / null-byte columns described by `desc`, to the host
int  sort_copy_rows(SortState* s, uint8_t* const* vals, uint8_t* const* nulls, const std::vector<ColRef>& desc, const uint32_t* perm_dev, int64_t n,
                    int64_t skip, cudaStream_t stream, std::vector<SortOutCol>& out, std::string& err);
// dst[i] = src[perm[i]] for one value / null-byte column of type `prim` (device)
int  sort_gather_rows(SortState* s, const uint8_t* src_vals, const uint8_t* src_null, int prim, const uint32_t* perm_dev, int64_t n,
                      uint8_t* dst_vals, uint8_t* dst_null, cudaStream_t stream);
void sort_close(SortState* s);

}  // namespace bk

// sort.h — K5 (ORDER BY / top-k) and K1 (filter-only stream compaction): host entry points used by api.cu.
// A SortState belongs to a plan: it allocates through the plan's allocator, runs on its stream and reports failures through
// bkgpu_plan::fail.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "../include/bkgpu.h"
#include "plan.h"
#include "prims.cuh"

namespace bk {

struct SortState;  // opaque (sort.cu)

struct SortOutCol {
    int tuple_id, slot_id, prim, elem;
    std::vector<uint8_t> values;
    std::vector<uint8_t> validity;  // LSB bitmap, empty = all valid
};

int  sort_open(bkgpu_plan* p, const Compiled& c, int64_t region_base, SortState** out);
int  sort_push(SortState* s, const DevCol* cols, int64_t nrows, bkgpu_stats* stats);
int  sort_finish(SortState* s, void* nccl_comm, int nranks, bkgpu_stats* stats, std::vector<SortOutCol>& out, int64_t* nrows);
size_t sort_partial_bytes(SortState* s);
int  sort_partial_export(SortState* s, void* dev_dst);
int  sort_partial_merge(SortState* s, const void* dev_src, int nranks, std::vector<SortOutCol>& out, int64_t* nrows);
void sort_reset(SortState* s);

// ---- the window stage (window.cu) over a SortState's retained rows (a PK_WINDOW plan retains its filtered rows like a full sort) ----
RowStore& sort_retained(SortState* s);
// stable LSD radix sort of the row ids `ids` (device, n entries, the current order) by `keys`; key k's image is output keys[k].out_reg
// of program progs[k] over `cols`
int  sort_stable_ids(SortState* s, const DevCol* cols, int64_t n, const std::vector<SortKey>& keys, const std::vector<const Program*>& progs,
                     uint32_t* ids, bkgpu_stats* stats);
void sort_close(SortState* s);

}  // namespace bk

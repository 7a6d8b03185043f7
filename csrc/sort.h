// sort.h — K5 (ORDER BY / top-k) and K1 (filter-only stream compaction): host entry points of the sort stage.
// A SortState belongs to a plan: it allocates through the plan's allocator, runs on its stream, reports failures through
// bkgpu_plan::fail and writes its rows into the plan's result.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <functional>
#include <vector>
#include "../include/bkgpu.h"
#include "plan.h"
#include "prims.cuh"

namespace bk {

struct SortState;  // opaque (sort.cu)

// `c` belongs to the plan and outlives the state
int  sort_open(bkgpu_plan* p, const Compiled& c, int64_t region_base, SortState** out);
int  sort_push(SortState* s, const DevCol* cols, int64_t nrows, bkgpu_stats* stats);
// n rows produced on the device into a post fragment: its input columns get room for n rows (`cap` when they grow), `fill` writes their
// values and null bytes, then they are packed (CTAs: grid_for(…, p->sm_count, per_sm)) and pushed, the push counting into `stats`
int  sort_feed(SortState* s, int64_t n, int64_t cap, int per_sm, bkgpu_stats* stats, const std::function<int(RowStore& in)>& fill);
// the fragment's rows into p->result; `desc`: their output column descriptions (nullptr = the fragment's own columns, kind 0)
int  sort_finish(SortState* s, void* nccl_comm, int nranks, bkgpu_stats* stats, const OutCol* desc);
size_t sort_partial_bytes(SortState* s);
int  sort_partial_export(SortState* s, void* dev_dst);
int  sort_partial_merge(SortState* s, const void* dev_src, int nranks);   // and the merged rows into p->result
void sort_reset(SortState* s);

// ---- the window stage (window.cu) over a SortState's retained rows (a PK_WINDOW plan retains its filtered rows like a full sort) ----
RowStore& sort_retained(SortState* s);
// stable LSD radix sort of the row ids `ids` (device, n entries, the current order) by `keys`; key k's image is output keys[k].out_reg
// of program progs[k] over `cols`
int  sort_stable_ids(SortState* s, const DevCol* cols, int64_t n, const std::vector<SortKey>& keys, const std::vector<const Program*>& progs,
                     uint32_t* ids, bkgpu_stats* stats);
void sort_close(SortState* s);

}  // namespace bk

// rb.h — rb_build_agg: the device build of per-group Roaring bitmaps from the pair buffer (rb.cu)
#pragma once
#include <stdint.h>
#include <vector>
#include "dev_types.h"
#include "prims.cuh"

struct bkgpu_plan;

namespace bk {

struct RbState {
    uint64_t* keys = nullptr;                          // the pair buffer (AggArgs::rb_keys), `cap` keys + 1
    unsigned long long* ctr = nullptr;                 // keys appended to it (AggArgs::rb_ctr)
    uint64_t cap = 0;
    uint64_t hi = 0;                                   // upper bound of the keys it holds (exact after a compaction)
    uint64_t* alt = nullptr;                           // the radix sort's second buffer, as large as the pair buffer
    RadixScratch sort;                                 // the radix sort's scratch, grow-only
    void* scratch[14] = {}; size_t scratch_cap[14] = {};   // grow-only device scratch of the build
    // the finished bitmaps of a request: ids (slot << 2 | rb_idx, ascending), offsets into `bytes` (one more than ids)
    std::vector<uint32_t> bid;
    std::vector<uint64_t> off;
    uint8_t* bytes = nullptr; size_t bytes_cap = 0;    // pinned, grow-only: the device-to-host copy runs at the link's speed
    // per rb_build_agg, its result column as bkgpu_get_next hands it out (rows + 1 int64 offsets, then the bytes); kept across requests,
    // so a re-armed plan writes into memory it has touched before
    std::vector<uint8_t> col[MAX_RB];
};

// sort and deduplicate the pair buffer in place; *n_out = the distinct keys it now holds (the device counter is set to it).
// BKGPU_ETOOBIG (naming rb_pair_capacity) when keys were already lost to a full buffer
int rb_compact(bkgpu_plan* p, uint64_t* n_out);
// after the request's last launch: compacts, builds and serializes every (group, rb_build_agg) bitmap on the device and copies the
// bytes and their directory into p->agg.rb
int rb_build(bkgpu_plan* p);

}  // namespace bk

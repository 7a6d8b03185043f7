// apply.cu — a scalar subquery under an aggregate (Compiled::sub; plan.cpp::lower_scalar_apply): the subquery's aggregate grouped by its
// correlation keys fills a second group table (bkgpu_plan::sub_agg); every outer batch is then looked up in it, chunk by chunk, by
// k_apply_lookup, which writes each referenced aggregate's finalized value as a typed column, and the plan's aggregate runs over the outer
// columns and those (launch_agg_batch: lean, direct or interpreter, as for any other batch).
#include <string.h>
#include <algorithm>
#include "api_state.h"
#include "dev_common.cuh"
#include "prims.cuh"

namespace bk {

// the lookup of one chunk of outer rows
struct LookupArgs {
    GroupTable gt;                 // the subquery's table (read only)
    AggPlan ap;                    // ... and its plan: the key packing and the aggregates
    DevCol keys[MAX_GROUP];        // the outer key columns, in the order of the subquery's keys
    int32_t n_out;
    int32_t out_agg[MAX_AGG];      // per output column: the subquery aggregate (index into ap.agg)
    int32_t out_stype[MAX_AGG];
    void* out_vals[MAX_AGG];
    uint32_t* out_valid[MAX_AGG];  // validity bitmaps, one 32-bit word per warp tile of 32 rows
    int64_t nrows;
};

// whether a group's key equals row `row`'s outer values, and its slot in *slot: the key is packed as lower_agg packs the subquery's
// group key (the same words, the same casts) and found with table_upsert's hash and linear probing, without inserting.  A NULL outer value
// never equals anything, so it finds no group — and the NULL-key group, whose null-flag bit no packed outer key has, is never found
__device__ __forceinline__ bool find_group(const LookupArgs& a, int64_t row, uint32_t* found_slot) {
    const AggPlan& ap = a.ap;
    uint64_t key[MAX_KEYW];
    for (int w = 0; w < ap.n_keyw; w++) key[w] = 0;
    for (int g = 0; g < ap.n_group; g++) {
        const DevCol& c = a.keys[g];
        if (elem_is_null(c, row)) return false;
        const uint64_t v = cast_prim(load_elem(c, row), c.prim, ap.key_prim[g]);
        const uint64_t m = ap.key_bits[g] >= 64 ? ~0ull : ((1ull << ap.key_bits[g]) - 1ull);
        key[ap.key_word[g]] |= (v & m) << ap.key_shift[g];
    }
    const GroupTable& gt = a.gt;
    uint32_t slot = (ap.n_keyw == 1 ? hash_key1(key[0]) : hash_key(key, ap.n_keyw)) & gt.cap_mask;
    const uint32_t cap = gt.cap_mask + 1;
    for (uint32_t probes = 0; probes < cap; probes++) {
        const uint32_t s = __ldg(gt.state + slot);
        if (s == 0u) return false;   // (the table is complete: no slot is busy)
        bool same = true;
        for (int w = 0; w < ap.n_keyw && same; w++) same = __ldg((const unsigned long long*)gt.keys + (size_t)w * cap + slot) == key[w];
        if (same) { *found_slot = slot; return true; }
        slot = (slot + 1) & gt.cap_mask;
    }
    return false;
}

__global__ void __launch_bounds__(256) k_apply_lookup(const __grid_constant__ LookupArgs a) {
    const AggPlan& ap = a.ap;
    const int lane = threadIdx.x & 31;
    const uint32_t cap = a.gt.cap_mask + 1;
    // warp-uniform tiles of 32 rows: each output column's 32 validity bits are one ballot and one store
    for (int64_t w0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); w0 < a.nrows; w0 += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = w0 + lane;
        const bool live = row < a.nrows;
        uint32_t slot = 0;
        const bool found = live && find_group(a, row, &slot);
        for (int k = 0; k < a.n_out; k++) {
            const AggSpec s = ap.agg[a.out_agg[k]];
            // finalized as extract_group does; no group: the empty-input row of a scalar AGG (COUNT 0, everything else NULL)
            uint64_t v = 0;
            bool valid = s.kind == AG_COUNT_STAR || s.kind == AG_COUNT;
            if (found) {
                // (only the lanes this aggregate finalizes from: one random load each)
                const bool need_cnt = s.kind != AG_COUNT_STAR, need_acc = need_cnt && s.kind != AG_COUNT;
                const uint64_t cnt = need_cnt && s.cnt_lane < ap.n_lanes ? __ldg((const unsigned long long*)a.gt.lanes + (size_t)s.cnt_lane * cap + slot) : 0;
                const uint64_t acc = need_acc && s.acc_lane < ap.n_lanes ? __ldg((const unsigned long long*)a.gt.lanes + (size_t)s.acc_lane * cap + slot) : 0;
                switch (s.kind) {
                    case AG_COUNT_STAR: v = __ldg((const unsigned long long*)a.gt.lanes + slot); break;   // (lane 0: the group's row count)
                    case AG_COUNT: v = cnt; break;
                    case AG_AVG: valid = cnt != 0; if (valid) v = f64_bits(__ddiv_rn(__dadd_rn(bits_f64(acc), 0.0), (double)(int64_t)cnt)); break;
                    default: valid = cnt != 0; if (valid) v = acc; break;   // SUM in its lane class, MIN / MAX in the argument's
                }
            }
            if (live) {
                switch (a.out_stype[k]) {
                    case ST_I32: ((int32_t*)a.out_vals[k])[row] = (int32_t)(int64_t)v; break;
                    case ST_U32: ((uint32_t*)a.out_vals[k])[row] = (uint32_t)v; break;
                    case ST_F32: ((float*)a.out_vals[k])[row] = (float)bits_f64(v); break;
                    case ST_U8: ((uint8_t*)a.out_vals[k])[row] = v ? 1 : 0; break;
                    default: ((uint64_t*)a.out_vals[k])[row] = v; break;
                }
            }
            const uint32_t bits = __ballot_sync(0xFFFFFFFFu, live && valid);
            if (lane == 0) a.out_valid[k][w0 >> 5] = bits;
        }
    }
}

}  // namespace bk

// ------------------------------------------------------------------------------------------
// host path
// ------------------------------------------------------------------------------------------
int apply_open(bkgpu_plan* p) {
    AggState* g = new AggState();
    p->sub_agg = g;
    const AggState& o = p->agg;   // (the plan's options are the aggregate's)
    g->env = o.env; g->group_cap_log2 = o.group_cap_log2; g->partial_cap = o.partial_cap; g->hll_cap = o.hll_cap; g->rb_cap = o.rb_cap;
    g->blocking_sync = o.blocking_sync;
    g->lookup_only = true; g->table_name = "the scalar subquery's group table";
    return agg_open(p, *g, *p->c.sub);
}

static int sub_batch(bkgpu_plan* p, const DevCol* cols, int64_t nrows, int64_t, bool vec_ok) {
    return launch_agg_batch(p, *p->sub_agg, *p->c.sub, cols, nrows, vec_ok);
}

// one outer batch (its columns in ApplyState::outer_want order): the lookup, then the aggregate, a chunk at a time so that the looked-up
// columns stay bounded
static int outer_batch(bkgpu_plan* p, const DevCol* cols, int64_t nrows, int64_t, bool vec_ok) {
    const Compiled& c = p->c;
    const Compiled& s = *c.sub;
    ApplyState& st = p->apply;
    const int64_t chunk = std::min<int64_t>(nrows, (int64_t)16 << 20);   // (a multiple of 32: every chunk's bitmaps start at a word)
    int rc;
    for (size_t k = 0; k < c.sub_out_cols.size(); k++)
        if ((rc = ensure_buf(p, &st.out_vals[k], &st.vals_cap[k], (size_t)chunk * 8)) || (rc = ensure_buf(p, &st.out_valid[k], &st.valid_cap[k], (size_t)chunk / 8 + 8)))
            return rc;
    LookupArgs a; memset(&a, 0, sizeof a);
    a.gt = p->sub_agg->gt; a.ap = s.ap;
    a.n_out = (int)c.sub_out_cols.size();
    for (int k = 0; k < a.n_out; k++) {
        a.out_agg[k] = c.sub_out_agg[(size_t)k];
        a.out_stype[k] = prim_storage(c.cols[(size_t)c.sub_out_cols[(size_t)k]].prim);
        a.out_vals[k] = st.out_vals[k]; a.out_valid[k] = (uint32_t*)st.out_valid[k];
    }
    std::vector<DevCol> all(c.cols.size());
    for (int64_t off = 0; off < nrows; off += chunk) {
        const int64_t n = std::min(chunk, nrows - off);
        for (size_t i = 0; i < st.outer_map.size(); i++) all[(size_t)st.outer_map[i]] = col_at(cols[i], off);
        for (int k = 0; k < a.n_out; k++) {
            DevCol& d = all[(size_t)c.sub_out_cols[(size_t)k]];
            d.values = st.out_vals[k]; d.validity = (const uint8_t*)st.out_valid[k];
            d.prim = c.cols[(size_t)c.sub_out_cols[(size_t)k]].prim; d.stype = prim_storage(d.prim);
        }
        for (size_t g = 0; g < c.sub_key_cols.size(); g++) a.keys[g] = all[(size_t)c.sub_key_cols[g]];
        a.nrows = n;
        k_apply_lookup<<<grid_for(n, p->sm_count, 8), 256, 0, p->stream>>>(a);
        CK(p, cudaGetLastError());
        p->stats.kernel_launches++;
        if ((rc = launch_agg_batch(p, p->agg, c, all.data(), n, vec_ok))) return rc;
    }
    return BKGPU_OK;
}

// a batch belongs to the subquery when its columns name the subquery's scan tuple; every subquery batch comes before the first outer batch
int apply_push(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    const Compiled& c = p->c;
    const Compiled& s = *c.sub;
    ApplyState& st = p->apply;
    bool is_sub = false;
    for (int k = 0; k < ncols; k++) is_sub = is_sub || cols[k].tuple_id == s.scan_tuple;
    int rc;
    if (is_sub) {
        if (st.outer_started)
            return p->fail(BKGPU_ESTATE, "a batch of the scalar subquery's tuple %d arrived after the first outer batch (every outer row looks up the whole "
                           "subquery's table)", s.scan_tuple);
        if ((rc = feed(p, s.cols, cols, ncols, nrows, on_device, sub_batch))) return rc;
        return learn_groups_async(p, *p->sub_agg, s);
    }
    if (st.outer_want.empty())
        for (size_t i = 0; i < c.cols.size(); i++)
            if (c.cols[i].tuple_id == c.scan_tuple) { st.outer_want.push_back(c.cols[i]); st.outer_map.push_back((int)i); }
    st.outer_started = true;
    if ((rc = feed(p, st.outer_want, cols, ncols, nrows, on_device, outer_batch))) return rc;
    return learn_groups_async(p, p->agg, c);
}

int apply_finish(bkgpu_plan* p) {
    AggState& g = *p->sub_agg;
    uint32_t local[8];
    uint32_t* ctr = g.h_pinned ? g.h_pinned + 8 : local;
    CK(p, cudaMemcpyAsync(ctr, g.gt.n_groups, 32, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    p->stats.d2h_bytes += 32;
    uint32_t copy[8];
    memcpy(copy, ctr, sizeof copy);
    return agg_take_counters(p, g, copy);
}

int apply_reset(bkgpu_plan* p) {
    p->apply.outer_started = false;
    return agg_reset(p, *p->sub_agg, *p->c.sub);
}

void apply_close(bkgpu_plan* p) {
    if (!p->sub_agg) return;
    agg_close(*p->sub_agg);
    delete p->sub_agg;
    p->sub_agg = nullptr;
}

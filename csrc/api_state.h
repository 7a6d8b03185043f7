// api_state.h — the plan object behind the C ABI (bkgpu_plan), the state of its hash join (JoinState, join.cu) and of its aggregate
// (AggState, agg.cu), and the host helpers the stages share.  ORDER BY / filter / window retention and the post fragment each keep a
// SortState (sort.cu).  bkgpu_plan itself holds what more than one stage uses: the compiled plan, the device, streams and lifecycle
// state, the staging buffers, the result, the stats and the allocator.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <time.h>
#include <atomic>
#include <string>
#include <vector>
#include "../include/bkgpu.h"
#include "agg_select.h"
#include "plan.h"
#include "sort.h"
#include "window.h"
#include "rb.h"

using namespace bk;

namespace bk {

enum State { S_INIT = 0, S_OPEN = 1, S_FINISHED = 2, S_CLOSED = 3 };

struct HostCol {  // one materialised result column (host memory owned by the plan)
    OutCol desc;
    int elem = 0;
    std::vector<uint8_t> values;
    std::vector<uint8_t> validity;  // LSB bitmap; empty = all valid
    const std::vector<uint8_t>* varlen = nullptr;   // elem < 0 (BITMAP): the whole column, rows + 1 int64 offsets then the bytes
    std::vector<uint8_t> batch;     // elem < 0: a later bkgpu_get_next batch, re-based (n + 1 offsets from 0, then its bytes)
};

struct EventPair { cudaEvent_t a, b; int64_t bytes; };

// FK -> PK join fast path: unique build keys, looked up through a dense array (small key range) or a packed
// (key32 << 32 | row) table; build-side columns are gathered to probe-row alignment
struct JoinFast {
    int32_t mode;               // 0 = none, 1 = dense array, 2 = packed 32-bit-key table
    const uint32_t* dense; uint64_t dense_min; uint64_t dense_size; uint64_t bias;
    const uint64_t* packed; uint32_t packed_mask;
};

// one retained build side of a hash join (K4) and its key indexes
struct JoinSide {
    RowStore store;   // the table's rows, by plan column (this side's columns only)
    uint8_t* keybits = nullptr; size_t keybits_cap = 0;   // validity of the build key AND the dimension's (star) / build child's (two-table) own filter
    uint64_t* jt_keys = nullptr; uint32_t* jt_rows = nullptr; uint32_t jt_mask = 0; bool jt_generic = false;   // multimap (duplicate keys)
    JoinFast jf{}; uint32_t* jf_dense = nullptr; uint64_t* jf_packed = nullptr; size_t jf_dense_cap = 0, jf_packed_cap = 0;   // unique-key index
    bool learned = false; uint64_t learn_min = 0, learn_max = 0;   // key range of the side's previous build (skips the min/max pass + round trip)
};

// the hash join (K4) of a plan (join.cu): retained build sides, their indexes, the probe's buffers.  Buffers and indexes are kept
// across bkgpu_reset; join_reset clears what belongs to one request.
struct JoinState {
    JoinSide side[4];            // the two-table join uses side[0], a star join one per dimension
    bool built = false;          // the build side is complete and indexed: probe batches have started
    bool tail_launch = false;    // the aggregate launch in progress is the outer-join tail (join_tail)
    std::vector<ColRef> probe_want; std::vector<int> probe_map;   // probe-side columns and their index in c.cols
    uint64_t* scratch = nullptr; size_t scratch_cap = 0;   // [0..1] key min / max, then u32 flags: [4] duplicate build key, [5] fused probe unusable, [6] key outside the learned range
    JoinProbe jp{}; int jp_key_pos = 0;   // the FK -> PK probe fused into the lean aggregate
    uint32_t* jp_attr = nullptr; uint64_t* jp_packed = nullptr; size_t jp_attr_cap = 0, jp_packed_cap = 0;
    uint8_t* matched = nullptr; size_t matched_cap = 0;   // LEFT / SEMI / ANTI: build rows that found a partner (1), or that the build child's filter removed (2)
    uint8_t* probe_bits = nullptr; size_t probe_bits_cap = 0;   // the probe key's validity AND the probe child's own filter, for one probe batch
    uint32_t* pairs = nullptr; size_t pairs_cap = 0;   // PK_JOIN, FULL: (probe row, build row) pairs of one batch
    uint32_t* cursor = nullptr; size_t cursor_cap = 0;   // the count of a pass: pairs, the FK -> PK gather's misses, the star probe's survivors
    uint32_t* tuples[2] = {nullptr, nullptr}; size_t tuples_cap[2] = {0, 0};   // star join: row-id tuples of one chunk (probe / expansion ping-pong)
    RowStore chunk;   // the gathered chunk (two-table gather path, FULL join under an aggregate, star join), by plan column
    // options
    int no_fused_probe = 0;
    int star_expand_cap = 0;     // test option "star_expand_capacity": first capacity (tuples) of a star join's expansion pass (0 = twice its input)
};

// the aggregate of a plan (agg.cu): its group table, the exchange between ranks, the extraction of the result, what earlier requests taught
// it, and its options.  Buffers are kept across bkgpu_reset; agg_reset clears what belongs to one request.
struct AggState {
    GroupTable gt{};
    uint64_t* d_rows_passed = nullptr;   // the table's counter block: [4..5] rows that passed the filter
    uint32_t* d_cursor = nullptr;        // ... [2] result cursor, [3] merge info (the largest group count of any rank)
    // the exchange between ranks
    uint64_t* d_partial = nullptr;  // export buffer (this rank)
    uint64_t* d_gather = nullptr;   // nranks export buffers
    size_t d_partial_cap = 0, d_gather_cap = 0;
    uint32_t merge_bound = 0, merge_bound_used = 0;   // groups per rank the all-gather is sized for (learned from earlier runs)
    uint32_t* d_part_cursors = nullptr;               // hash repartition of the groups across ranks (option "repartition")
    int rank = -1;                // this rank in the communicator (-1 = not asked yet; the all-gather merge skips its own rows)
    // extraction: device buffers (kept across resets) and their pinned landing area
    uint64_t* d_outv = nullptr; uint8_t* d_outn = nullptr; size_t out_cap_alloc = 0;
    uint64_t* h_outv = nullptr; uint8_t* h_outn = nullptr; size_t h_out_cap = 0;
    // mapped host buffer the lean kernel's last CTA extracts the result into (AggArgs::fused_out), and whether the request's last
    // aggregate launch did so: then agg_finish only waits and reads it
    uint8_t* h_fused = nullptr; uint8_t* d_fused = nullptr; size_t fused_bytes = 0; uint32_t fused_cap = 0; bool fused_last = false;
    // learned
    uint32_t* h_pinned = nullptr;   // [0] groups seen (async copy after every aggregate launch that does not extract its result), [8..15] counter block; pinned
    uint32_t known_groups = 0;
    int64_t finish_groups = -1;     // groups in the table when the last finish read the result back (-1 = unknown: full re-initialisation)
    int fx_off = 0;                 // set when a finished request saw more than 1/64 of its surviving rows take FX's exact path (see agg_take_counters)
    uint64_t rows_passed_host = 0;
    bool blocking_wait = false; cudaEvent_t wait_event = nullptr;   // see agg_wait
    std::vector<uint8_t> hll_host;   // the HLL arena's claimed blocks, copied back by a finished request (agg_result reads the sketches there)
    RbState rb;                      // rb_build_agg's pair buffer and build (rb.h)
    // options: what the kernel choice reads (bkgpu_set_option writes them; launch_agg_batch fills in the per-launch fields of a copy).  By
    // default COUNT(*) WHERE int32 <cmp> c runs the TMA-staged kernel (scalar_tma.cu), and the lean kernel's double sums are fixed-point
    // limbs (FX, agg_direct.cuh) unless the environment's BKGPU_LEAN_FX says otherwise
    AggEnv env = [] { AggEnv e; e.scalar_tma = 1; const char* v = getenv("BKGPU_LEAN_FX"); e.lean_fx = v ? atoi(v) != 0 : BK_LEAN_FX_DEFAULT; return e; }();
    int group_cap_log2 = 20;
    int64_t partial_cap = 1 << 16;
    int64_t hll_cap = 4096;          // option hll_group_capacity: sketches the register arena holds (16 KB each: 64 MB by default)
    int64_t rb_cap = (int64_t)1 << 27;   // option rb_pair_capacity: keys the rb_build_agg pair buffer holds (8 bytes each, twice: the sort's buffers)
    int repartition = 0;
    int blocking_sync = -1;
};

// BKGPU_TRACE=1: wall-clock time the HOST spends in each phase of a request (summed per plan, printed by bkgpu_close)
struct HostClock {
    double reset = 0, push = 0, collective = 0, extract_wait = 0, finish = 0; int64_t n = 0;
    static double now() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec / 1e6; }
};

}  // namespace bk

extern thread_local std::string g_thread_error;

struct bkgpu_plan {
    Compiled c;
    int device = 0;
    int sm_count = 132;
    State state = S_INIT;
    std::string last_error;
    std::atomic<int> cancelled{0};
    void* nccl_comm = nullptr;
    int nranks = 1;
    // options
    cudaStream_t stream = nullptr; bool own_stream = false;
    cudaStream_t copy_stream = nullptr;
    int64_t batch_capacity = 1 << 20;
    int64_t chunk_rows = 8 << 20;
    int64_t region_base = 0;      // arrival index of this plan's first row (ties across GPUs break by (region, row))
    HostClock hclk; bool trace = getenv("BKGPU_TRACE") != nullptr;
    // host staging for pageable / pinned pushes
    std::vector<void*> stage[2];
    std::vector<void*> stage_valid[2];
    size_t stage_rows = 0;
    cudaEvent_t stage_free[2] = {nullptr, nullptr}, stage_ready[2] = {nullptr, nullptr};
    std::vector<uint8_t*> bounce[2]; size_t bounce_rows = 0; cudaEvent_t bounce_done[2] = {nullptr, nullptr}; bool bounce_busy[2] = {false, false};
    // the stages
    SortState* sort = nullptr;        // ORDER BY / filter / window retention (PK_SORT, PK_FILTER, PK_WINDOW)
    SortState* post = nullptr;        // the post fragment (Compiled::post) above an aggregate, a window or a join that returns rows: above an
                                      // aggregate, its sort / HAVING, or the input rows of its window stages
    SortState* outer = nullptr;       // windows above an aggregate: the query's ORDER BY over the window rows (Compiled::post->post)
    JoinState join;                   // hash join (K4): PK_JOIN_AGG, PK_JOIN, PK_STAR_AGG
    AggState agg;                     // the aggregate: PK_AGG, PK_JOIN_AGG, PK_STAR_AGG
    // results
    std::vector<HostCol> result;
    int64_t result_rows = 0, result_pos = 0;
    // stats
    bkgpu_stats stats{};
    std::vector<EventPair> timed;
    std::vector<EventPair> timed_coll;
    std::vector<cudaEvent_t> event_pool;
    std::vector<std::pair<void*, size_t>> dev_allocs;   // (buffer, size class) — returned to the process-wide cache on free / close

    int fail(int code, const char* fmt, ...) {
        char buf[512]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
        last_error = buf; g_thread_error = buf; return code;
    }
    int cuda_fail(cudaError_t e, const char* what) {
        return fail(e == cudaErrorMemoryAllocation ? BKGPU_ENOMEM : BKGPU_ENODEV, "%s: %s", what, cudaGetErrorString(e));
    }
};

#define CK(plan, call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return (plan)->cuda_fail(e__, #call); } while (0)

// ---- api.cu
// device buffers from the process-wide cache; ensure_buf: grow-only (plans are re-armed with bkgpu_reset and run again)
int dev_alloc(bkgpu_plan* p, void** out, size_t bytes);
void dev_free(bkgpu_plan* p, void* ptr);
int ensure_buf(bkgpu_plan* p, void** ptr, size_t* cap, size_t bytes);
// mapped host buffers of the fused extraction, kept in a process-wide cache by size: take = nullptr when none is free, put = false when the
// cache does not keep it (the caller frees it)
uint8_t* mapped_take(size_t bytes);
bool mapped_put(size_t bytes, uint8_t* buf);
int cpu_budget();   // CPUs this process may use (affinity, cgroup quota)
// device buffers of one call: returned to the plan's allocator when the scope ends, on every way out of the call
struct DevScope {
    bkgpu_plan* p;
    std::vector<void*> bufs;
    explicit DevScope(bkgpu_plan* plan) : p(plan) {}
    DevScope(const DevScope&) = delete;
    DevScope& operator=(const DevScope&) = delete;
    ~DevScope() { for (void* b : bufs) dev_free(p, b); }
    template <class T> int alloc(T** out, size_t bytes) {
        const int rc = dev_alloc(p, (void**)out, bytes);
        if (rc == BKGPU_OK) bufs.push_back(*out);
        return rc;
    }
    void release(void* b) {   // before the scope ends
        for (auto it = bufs.begin(); it != bufs.end(); ++it) if (*it == b) { bufs.erase(it); dev_free(p, b); return; }
    }
};
// a stage timer's two events, destroyed on every way out of the scope that holds them
struct StageTimer {
    cudaEvent_t a = nullptr, b = nullptr;
    StageTimer() { cudaEventCreate(&a); cudaEventCreate(&b); }
    StageTimer(const StageTimer&) = delete;
    StageTimer& operator=(const StageTimer&) = delete;
    ~StageTimer() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
};
// the plan's columns `want` resolved against one pushed batch
int bind_columns(bkgpu_plan* p, const std::vector<ColRef>& want, const bkgpu_column* cols, int ncols, int64_t nrows, std::vector<const bkgpu_column*>& bound);
// a batch as device columns (host columns chunk by chunk through the staging buffers), handed to `fn`
typedef int (*BatchFn)(bkgpu_plan*, const DevCol*, int64_t nrows, int64_t row_base, bool vec_ok);
int feed(bkgpu_plan* p, const std::vector<ColRef>& want, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device, BatchFn fn);

// rows [off, ...) of a device column
inline DevCol col_at(const DevCol& c, int64_t off) {
    DevCol x = c;
    x.values = (const uint8_t*)c.values + (size_t)off * (size_t)storage_bytes(c.stype);
    if (c.validity) x.validity = c.validity + off / 8;
    return x;
}

// ---- agg.cu: the aggregate (PK_AGG, PK_JOIN_AGG, PK_STAR_AGG)
int agg_open(bkgpu_plan* p);     // bkgpu_open: the group table and the pinned counter words (and the HLL arena, the rb_build_agg pair buffer)
int agg_push(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device);   // a PK_AGG batch
// the aggregate of `c` over one batch; `jp`: fused FK -> PK probe (lean kernel only), +1 without launching when the batch does not fit it
int launch_agg_batch(bkgpu_plan* p, const Compiled& c, const DevCol* cols, int64_t nrows, bool vec_ok, const JoinProbe* jp = nullptr);
int agg_finish(bkgpu_plan* p);   // the cross-rank merge (with a communicator), then the result and stats.rows_filtered
int agg_reset(bkgpu_plan* p);    // bkgpu_reset: the table is empty again
void agg_close(bkgpu_plan* p);   // bkgpu_close, once the plan's streams have drained: the host memory the aggregate holds
size_t agg_partial_bytes(const bkgpu_plan* p);
int agg_partial_export(bkgpu_plan* p, void* dev_dst);
int agg_partial_merge(bkgpu_plan* p, const void* dev_src, int nranks);   // and the result from the merged table

// ---- join.cu
int join_push(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device);   // PK_JOIN_AGG, PK_JOIN, PK_STAR_AGG
int join_tail(bkgpu_plan* p);    // LEFT / SEMI / ANTI_SEMI, after the last probe batch: the preserved rows the join type asks for
void join_reset(bkgpu_plan* p);  // bkgpu_reset: the next request retains its build sides afresh
JoinArgs join_args(const bkgpu_plan* p, bool tail);   // the general probe of the two-table join, as the aggregate kernels read it

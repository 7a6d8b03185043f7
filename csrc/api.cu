// api.cu — the C ABI of include/bkgpu.h: plan lifecycle (ExecNode::init/open/get_next/close
// inverted into init/open/push/finish/get_next/close), batch staging, the aggregate's launch, exchange and result materialisation.
// The hash join's host path is join.cu; the plan object (bkgpu_plan) is api_state.h.
#include <dlfcn.h>
#include <sched.h>
#include <string.h>
#include <algorithm>
#include <condition_variable>
#include <functional>
#include <map>
#include <mutex>
#include <thread>
#include "api_state.h"
#include "hll.cuh"
#include "nccl_dl.h"
#include "prims.cuh"
#include "build_id.h"

thread_local std::string g_thread_error;

static int thread_fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    g_thread_error = buf;
    return code;
}

// ------------------------------------------------------------------ library
extern "C" const char* bkgpu_version(void) { return "bkgpu 0.2 (sm_90a) src=" BKGPU_SRC_DIGEST; }   // digest of csrc/ + include/ at compile time (csrc/Makefile)

extern "C" int bkgpu_device_count(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) { g_thread_error = std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e); return BKGPU_ENODEV; }
    return n;
}

extern "C" const char* bkgpu_last_error(bkgpu_plan* p) { return p ? p->last_error.c_str() : g_thread_error.c_str(); }

extern "C" int bkgpu_plan_explain(const uint8_t* desc, size_t len, char* text, size_t text_len) {
    Compiled c; std::string err;
    int rc = compile_plan(desc, len, c, err);
    if (rc != BKGPU_OK) { if (text && text_len) snprintf(text, text_len, "%s", err.c_str()); return thread_fail(rc, err.c_str()); }
    if (text && text_len) snprintf(text, text_len, "%s", c.explain.c_str());
    return BKGPU_OK;
}

// ------------------------------------------------------------------ helpers
// Device buffers come from a process-wide cache of freed buffers (per device, per size class): a store opens and closes one plan per
// request (the reference builds its ExecNode tree per request, src/store/region.cpp:3072), and cudaMalloc / cudaFree of the 40 MB group
// table cost milliseconds and a device-wide synchronisation each.  A buffer enters the cache only after the owning plan's streams have
// drained.  BKGPU_NO_ALLOC_CACHE=1 turns the cache off; bkgpu_release_cache() returns its memory to the driver.
namespace {
struct DevCache {
    std::mutex mu;
    std::multimap<std::pair<int, size_t>, void*> free_;
    size_t held = 0;
    const size_t limit = (size_t)8 << 30;
    const bool off = getenv("BKGPU_NO_ALLOC_CACHE") && atoi(getenv("BKGPU_NO_ALLOC_CACHE")) != 0;
    void* take(int device, size_t sc) {
        std::lock_guard<std::mutex> g(mu);
        auto it = free_.find({device, sc});
        if (it == free_.end()) return nullptr;
        void* q = it->second; free_.erase(it); held -= sc;
        return q;
    }
    bool put(int device, size_t sc, void* q) {
        std::lock_guard<std::mutex> g(mu);
        if (off || held + sc > limit) return false;
        free_.insert({{device, sc}, q}); held += sc;
        return true;
    }
    void release_all() {   // (the caller has the right device current for none of them: cudaFree takes any device's pointer)
        std::lock_guard<std::mutex> g(mu);
        for (auto& kv : free_) cudaFree(kv.second);
        free_.clear(); held = 0;
    }
};
DevCache& dev_cache() { static DevCache c; return c; }
// the mapped host buffers of the fused extraction (bkgpu_plan::h_fused) are kept the same way: pinning and unpinning one costs a
// plan's open and close about a tenth of a millisecond
struct MappedCache {
    std::mutex mu;
    std::multimap<size_t, uint8_t*> free_;
    uint8_t* take(size_t bytes) {
        std::lock_guard<std::mutex> g(mu);
        auto it = free_.find(bytes);
        if (it == free_.end()) return nullptr;
        uint8_t* q = it->second; free_.erase(it);
        return q;
    }
    bool put(size_t bytes, uint8_t* q) {
        std::lock_guard<std::mutex> g(mu);
        if (dev_cache().off || free_.size() >= 64) return false;
        free_.insert({bytes, q});
        return true;
    }
    void release_all() {
        std::lock_guard<std::mutex> g(mu);
        for (auto& kv : free_) cudaFreeHost(kv.second);
        free_.clear();
    }
};
MappedCache& mapped_cache() { static MappedCache c; return c; }
size_t size_class(size_t b) {   // eight classes per power of two: at most 12.5 % slack
    if (b < 256) return 256;
    size_t p2 = 1; while (p2 < b) p2 <<= 1;
    const size_t step = p2 >> 3;
    return (b + step - 1) / step * step;
}
}  // namespace
extern "C" void bkgpu_release_cache(void) { dev_cache().release_all(); mapped_cache().release_all(); }

int dev_alloc(bkgpu_plan* p, void** out, size_t bytes) {
    const size_t sc = size_class(bytes ? bytes : 8);
    void* q = dev_cache().take(p->device, sc);
    if (!q) {
        cudaError_t e = cudaMalloc(&q, sc);
        if (e != cudaSuccess) { cudaGetLastError(); dev_cache().release_all(); e = cudaMalloc(&q, sc); }   // memory held by the cache is memory the device has
        if (e != cudaSuccess) return p->cuda_fail(e, "cudaMalloc");
    }
    *out = q;
    p->dev_allocs.push_back({q, sc});
    return BKGPU_OK;
}
void dev_free(bkgpu_plan* p, void* ptr) {
    if (!ptr) return;
    size_t sc = 0;
    for (auto it = p->dev_allocs.begin(); it != p->dev_allocs.end(); ++it) if (it->first == ptr) { sc = it->second; p->dev_allocs.erase(it); break; }
    if (sc) {   // work queued on this plan's streams may still use the buffer
        if (p->stream) cudaStreamSynchronize(p->stream);
        if (p->copy_stream) cudaStreamSynchronize(p->copy_stream);
        if (dev_cache().put(p->device, sc, ptr)) return;
    }
    cudaFree(ptr);
}
// grow-only device buffer: plans are re-armed with bkgpu_reset and run again; cudaMalloc / cudaFree per run would
// serialise the device every time
int ensure_buf(bkgpu_plan* p, void** ptr, size_t* cap, size_t bytes) {
    if (*ptr && *cap >= bytes) return BKGPU_OK;
    dev_free(p, *ptr); *ptr = nullptr; *cap = 0;
    const int rc = dev_alloc(p, ptr, bytes);
    if (rc == BKGPU_OK) *cap = bytes;
    return rc;
}
// record = false: the caller records ep->a itself (right before its launch)
static EventPair* timer_begin(bkgpu_plan* p, std::vector<EventPair>& v, int64_t bytes, bool record = true) {
    EventPair ep{};
    for (cudaEvent_t* e : {&ep.a, &ep.b}) {   // events are recycled: a re-armed plan launches the same kernels again and again
        if (!p->event_pool.empty()) { *e = p->event_pool.back(); p->event_pool.pop_back(); }
        else if (cudaEventCreate(e) != cudaSuccess) return nullptr;
    }
    ep.bytes = bytes;
    if (record) cudaEventRecord(ep.a, p->stream);
    v.push_back(ep);
    return &v.back();
}
static void timer_end(bkgpu_plan* p, EventPair* ep) { if (ep) cudaEventRecord(ep->b, p->stream); }

// ------------------------------------------------------------------ lifecycle
extern "C" int bkgpu_init(bkgpu_plan** out, const uint8_t* desc, size_t len, int device, void* nccl_comm) {
    if (!out) return thread_fail(BKGPU_EINVAL, "bkgpu_init: out is NULL");
    *out = nullptr;
    bkgpu_plan* p = new bkgpu_plan();
    std::string err;
    int rc = compile_plan(desc, len, p->c, err);
    if (rc != BKGPU_OK) { g_thread_error = err; delete p; return rc; }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) {
        g_thread_error = std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") +
                         " (this library has no CPU fallback)";
        delete p; return BKGPU_ENODEV;
    }
    if (device < 0 || device >= ndev) { g_thread_error = "bkgpu_init: bad device index"; delete p; return BKGPU_EINVAL; }
    p->device = device;
    p->nccl_comm = nccl_comm;
    if (nccl_comm) {
        int n = 0;
        if (nccl_comm_count(nccl_comm, &n) != 0 || n < 1) { g_thread_error = std::string("NCCL: ") + nccl_last_error(); delete p; return BKGPU_ENCCL; }
        p->nranks = n;
    }
    { int n = 0; if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && n > 0) p->sm_count = n; }   // (cudaGetDeviceProperties costs milliseconds per call)
    *out = p;
    return BKGPU_OK;
}

extern "C" int bkgpu_set_option(bkgpu_plan* p, const char* key, int64_t v) {
    if (!p || !key) return thread_fail(BKGPU_EINVAL, "bkgpu_set_option: NULL argument");
    if (p->state != S_INIT) return p->fail(BKGPU_ESTATE, "options must be set before bkgpu_open");
    std::string k = key;
    if (k == "stream") { p->stream = (cudaStream_t)(uintptr_t)v; p->own_stream = false; }
    else if (k == "group_capacity_log2") { if (v < 4 || v > 30) return p->fail(BKGPU_EINVAL, "group_capacity_log2 out of range"); p->group_cap_log2 = (int)v; }
    else if (k == "smem_capacity_log2") { if (v < -1 || v > 13) return p->fail(BKGPU_EINVAL, "smem_capacity_log2 out of range"); p->smem_cap_log2 = (int)v; }
    else if (k == "batch_capacity") { if (v < 1) return p->fail(BKGPU_EINVAL, "batch_capacity must be positive"); p->batch_capacity = v; }
    else if (k == "chunk_rows") { if (v < 1024) return p->fail(BKGPU_EINVAL, "chunk_rows too small"); p->chunk_rows = (v + 7) & ~7ll; }
    else if (k == "rb_pair_capacity") { if (v < 1024 || v > RADIX_MAX_KEYS) return p->fail(BKGPU_EINVAL, "rb_pair_capacity out of range (1024 .. 2^30 - 1)"); p->rb_cap = v; }
    else if (k == "hll_group_capacity") { if (v < 1 || v > (1 << 20)) return p->fail(BKGPU_EINVAL, "hll_group_capacity out of range (1 .. 2^20)"); p->hll_cap = v; }
    else if (k == "partial_capacity") { if (v < 1) return p->fail(BKGPU_EINVAL, "partial_capacity must be positive"); p->partial_cap = v; }
    else if (k == "force_generic") p->force_generic = v != 0;
    else if (k == "lean_fx") p->lean_fx = v != 0;
    else if (k == "blocking_sync") p->blocking_sync = (int)v;
    else if (k == "star_expand_capacity") { if (v < 0 || v > 0x7FFFFFFF) return p->fail(BKGPU_EINVAL, "star_expand_capacity out of range"); p->join.star_expand_cap = (int)v; }
    else if (k == "no_lean") p->no_lean = v != 0;
    else if (k == "no_fused_probe") p->join.no_fused_probe = v != 0;
    else if (k == "repartition") p->repartition = v != 0;
    else if (k == "no_lean_nulls") p->no_lean_nulls = v != 0;
    else if (k == "no_lean_mm") p->no_lean_mm = v != 0;
    else if (k == "scalar_tma") p->scalar_tma = v != 0;
    else if (k == "region_base") p->region_base = v;
    else return p->fail(BKGPU_EINVAL, "unknown option '%s'", key);
    return BKGPU_OK;
}

static int alloc_group_table(bkgpu_plan* p) {
    const AggPlan& ap = p->c.ap;
    GroupTable& gt = p->gt;
    int log2 = ap.n_keyw == 0 ? 0 : p->group_cap_log2;
    size_t cap = (size_t)1 << log2;
    gt.cap_mask = (uint32_t)(cap - 1); gt.cap_log2 = (uint32_t)log2;
    int rc;
    if ((rc = dev_alloc(p, (void**)&gt.state, cap * 4))) return rc;
    if ((rc = dev_alloc(p, (void**)&gt.keys, cap * 8 * (size_t)std::max(ap.n_keyw, 1)))) return rc;
    if ((rc = dev_alloc(p, (void**)&gt.lanes, cap * 8 * (size_t)ap.n_lanes))) return rc;
    if ((rc = dev_alloc(p, (void**)&gt.n_groups, 4 * ((size_t)GT_OCC_OFF + cap)))) return rc;   // counter, overflow flag, occupied list
    gt.overflow = gt.n_groups + 1;
    if (ap.n_hll) {   // hll_add_agg: the register arena, one block per (group, sketch) that receives a value
        if ((rc = dev_alloc(p, (void**)&gt.hll_regs, (size_t)p->hll_cap * HLL_REGISTERS))) return rc;
        if ((rc = dev_alloc(p, (void**)&gt.hll_ctr, 16))) return rc;
        gt.hll_cap = (uint32_t)p->hll_cap;
        CK(p, cudaMemsetAsync(gt.hll_ctr, 0, 16, p->stream));
    }
    if (p->c.n_rb) {   // rb_build_agg: the pair buffer and the sort's second buffer (one word more each: the build's scan closes on it)
        if ((rc = dev_alloc(p, (void**)&p->rb.keys, ((size_t)p->rb_cap + 1) * 8))) return rc;
        if ((rc = dev_alloc(p, (void**)&p->rb.alt, ((size_t)p->rb_cap + 1) * 8))) return rc;
        if ((rc = dev_alloc(p, (void**)&p->rb.ctr, 8))) return rc;
        p->rb.cap = (uint64_t)p->rb_cap;
        CK(p, cudaMemsetAsync(p->rb.ctr, 0, 8, p->stream));
        p->rb.hi = 0;
    }
    p->d_cursor = gt.n_groups + 2;                       // [2] result cursor [3] merge info
    p->d_rows_passed = (uint64_t*)(gt.n_groups + 4);     // [4..5] rows that passed the filter
    CK(p, cudaMemsetAsync(gt.n_groups, 0, 4 * GT_OCC_OFF, p->stream));
    CK(p, launch_table_init(gt, ap, p->stream));
    p->stats.kernel_launches++;
    return BKGPU_OK;
}

namespace { int cpu_budget(); }   // CPUs this process may use (affinity, cgroup quota): defined with the copy pool

// the plan's IN sets (OP_IN_SET) in one device allocation, kept until bkgpu_close (bkgpu_reset keeps them), and their addresses
// patched into every program that probes them.  Part of opening the plan, not of a request: not counted in h2d_bytes.
static int upload_in_sets(bkgpu_plan* p) {
    if (!p->c.in_sets || p->c.in_sets->sets.empty()) return BKGPU_OK;
    const std::vector<InSet>& sets = p->c.in_sets->sets;
    size_t words = 0;
    for (const InSet& s : sets) words += s.image.size();
    uint64_t* d = nullptr;
    int rc = dev_alloc(p, (void**)&d, words * 8);
    if (rc) return rc;
    std::vector<uint64_t> addr;
    for (const InSet& s : sets) {
        addr.push_back((uint64_t)(uintptr_t)d);
        CK(p, cudaMemcpyAsync(d, s.image.data(), s.image.size() * 8, cudaMemcpyHostToDevice, p->stream));
        d += s.image.size();
    }
    CK(p, cudaStreamSynchronize(p->stream));
    patch_in_sets(p->c, addr);
    return BKGPU_OK;
}

extern "C" int bkgpu_open(bkgpu_plan* p) {
    if (!p) return thread_fail(BKGPU_EINVAL, "bkgpu_open: NULL plan");
    if (p->state != S_INIT) return p->fail(BKGPU_ESTATE, "bkgpu_open called twice");
    CK(p, cudaSetDevice(p->device));
    if (!p->stream) { CK(p, cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking)); p->own_stream = true; }
    CK(p, cudaStreamCreateWithFlags(&p->copy_stream, cudaStreamNonBlocking));
    if (cudaHostAlloc((void**)&p->h_pinned, 64, cudaHostAllocDefault) == cudaSuccess) memset(p->h_pinned, 0, 64); else p->h_pinned = nullptr;
    for (int i = 0; i < 2; i++) {
        CK(p, cudaEventCreateWithFlags(&p->stage_free[i], cudaEventDisableTiming));
        CK(p, cudaEventCreateWithFlags(&p->stage_ready[i], cudaEventDisableTiming));
    }
    p->blocking_wait = p->blocking_sync >= 0 ? p->blocking_sync != 0 : (p->nranks > 1 && cpu_budget() < 4 * p->nranks);
    if (p->c.ap.n_hll && p->repartition)
        return p->fail(BKGPU_EUNSUPPORTED, "hll_add_agg with the repartition merge is outside the GPU path: its sketches travel only with the all-gather of group rows");
    if (p->c.n_rb && p->nccl_comm)
        return p->fail(BKGPU_EUNSUPPORTED, "rb_build_agg with a communicator is outside the GPU path: bitmaps do not travel with the fixed-width partial rows");
    int rc = upload_in_sets(p);   // (before sort_open: it copies the programs)
    if (rc) return rc;
    if (p->c.kind == PK_AGG || p->c.kind == PK_JOIN_AGG || p->c.kind == PK_STAR_AGG) rc = alloc_group_table(p);
    if (!rc && (p->c.kind == PK_SORT || p->c.kind == PK_FILTER || p->c.kind == PK_WINDOW))   // (a window retains its rows like a full sort)
        rc = sort_open(p, p->c, p->region_base, &p->sort);
    if (!rc && p->c.post) { rc = sort_open(p, *p->c.post, 0, &p->post_sort); store_init(p->post, p->c.post->cols); }
    if (rc) return rc;
    p->state = S_OPEN;
    return BKGPU_OK;
}

// the group count an earlier launch left in pinned memory: the 4-byte copy after a launch, or the counter block of a fused extraction
// (read without a synchronisation: a stale value only costs speed)
static void learn_groups(bkgpu_plan* p) {
    if (p->h_pinned && p->h_pinned[0] > p->known_groups) p->known_groups = p->h_pinned[0];
    if (p->h_fused) { const uint32_t g = *(const volatile uint32_t*)p->h_fused; if (g > p->known_groups) p->known_groups = g; }
}

// device images of an extracted row: one per group expression, per aggregate its final value (+2 for an AVG blob)
static int agg_n_img(const AggPlan& ap) {
    int n = ap.n_group;
    for (int k = 0; k < ap.n_agg; k++) if (!ap.agg[k].hidden) n += ap.agg[k].kind == AG_AVG ? 3 : 1;
    return n;
}

// the mapped host buffer of the fused extraction, sized for the groups seen so far (at least 2048 rows); false = too many groups
// to extract this way (the table is then read back by k_extract)
static bool ensure_fused(bkgpu_plan* p) {
    uint32_t want = 2048;
    while (want < p->known_groups && want < (1u << 16)) want *= 2;
    if (want < p->known_groups) return false;
    if (p->h_fused && p->fused_cap >= want) return true;
    if (p->h_fused) {   // (a launch still running may write into it)
        cudaStreamSynchronize(p->stream);
        if (!mapped_cache().put(p->fused_bytes, p->h_fused)) cudaFreeHost(p->h_fused);
        p->h_fused = p->d_fused = nullptr; p->fused_cap = 0;
    }
    const size_t bytes = 32 + (size_t)want * (size_t)agg_n_img(p->c.ap) * 9;
    uint8_t* h = mapped_cache().take(bytes);
    if (!h && cudaHostAlloc((void**)&h, bytes, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return false; }
    if (cudaHostGetDevicePointer((void**)&p->d_fused, h, 0) != cudaSuccess) { cudaGetLastError(); cudaFreeHost(h); return false; }
    memset(h, 0, 32);
    p->h_fused = h; p->fused_bytes = bytes; p->fused_cap = want;
    return true;
}

// rb_build_agg: a launch appends at most one key per row and rb_build_agg aggregate, except where a probe row meets several build rows (such
// a launch can still overflow the pair buffer, and the request then fails at bkgpu_finish).  When the keys could outgrow the buffer, it is
// sorted and deduplicated first (a set does not depend on order), and the launch shrinks to the rows that fit
static int rb_room(bkgpu_plan* p, const Compiled& c, int64_t* rows) {
    const uint64_t per = (uint64_t)c.n_rb, cap = p->rb.cap;
    if (p->rb.hi + (uint64_t)*rows * per > cap) {
        uint64_t n = 0;
        const int rc = rb_compact(p, &n);
        if (rc) return rc;
        p->rb.hi = n;
        const int64_t fit = (int64_t)((cap - n) / per) & ~7ll;   // (a multiple of 8 rows: the next launch's validity bitmaps stay byte-aligned)
        if (fit < 8)
            return p->fail(BKGPU_ETOOBIG, "rb_build_agg: the pair buffer holds %llu distinct (group, value) pairs and is full: raise rb_pair_capacity",
                           (unsigned long long)n);
        if (*rows > fit && !p->join.tail_launch) *rows = fit;   // (the join's tail walks every build row in one launch)
    }
    p->rb.hi += (uint64_t)*rows * per;
    return BKGPU_OK;
}

int launch_agg_batch(bkgpu_plan* p, const Compiled& c, const DevCol* cols, int64_t nrows, bool vec_ok, const JoinProbe* jp) {
    AggEnv env;
    env.force_generic = p->force_generic; env.no_lean = p->no_lean; env.no_lean_nulls = p->no_lean_nulls; env.no_lean_mm = p->no_lean_mm;
    env.lean_fx = p->lean_fx; env.fx_off = p->fx_off;
    env.scalar_tma = p->scalar_tma; env.smem_cap_log2 = p->smem_cap_log2;
    env.tail_launch = p->join.tail_launch;
    env.multi_rank = p->nccl_comm && p->nranks > 1; env.has_post = p->c.post != nullptr;
    if (c.ap.n_keyw > 0 && p->smem_cap_log2 < 0) learn_groups(p);   // (the shared table is sized from it)
    env.known_groups = p->known_groups;
    AggArgs a; AggSelection sel;
    const int rc = select_agg_launch(c, cols, nrows, vec_ok, jp, env, a, sel);
    if (rc == BKGPU_ENOMEM) return p->fail(rc, "lean kernel: shared table does not fit");
    if (rc) return rc;
    a.gt = p->gt; a.rows_passed = p->d_rows_passed;
    if (c.kind == PK_JOIN_AGG) a.join = join_args(p, p->join.tail_launch);
    if (sel.fused_ok && ensure_fused(p)) { a.fused_out = p->d_fused; a.fused_cap = p->fused_cap; }
    const int64_t kMax = (int64_t)1 << 30;  // rows per launch (32-bit counters inside a CTA)
    int64_t algo_bytes_per_row = 0;
    for (int i = 0; i < a.n_cols; i++) algo_bytes_per_row += storage_bytes(a.cols[i].stype);
    int64_t b_rows = 0;
    for (int64_t off = 0; off < nrows; off += b_rows) {
        AggArgs b = a;
        b.nrows = std::min(kMax, nrows - off);
        if (c.n_rb) {   // (a compaction swaps the pair buffer with the sort's second buffer)
            const int rrc = rb_room(p, c, &b.nrows);
            if (rrc) return rrc;
            b.rb_keys = p->rb.keys; b.rb_ctr = p->rb.ctr; b.rb_cap = p->rb.cap;
        }
        b_rows = b.nrows;
        for (int i = 0; i < b.n_cols; i++) b.cols[i] = col_at(a.cols[i], off);
        EventPair* ep = timer_begin(p, p->timed, b.nrows * algo_bytes_per_row, false);
        cudaError_t e = launch_agg(b, sel.kernel, sel.smem, p->sm_count, p->stream, ep ? ep->a : nullptr);
        timer_end(p, ep);
        p->fused_last = b.fused_out != nullptr;
        if (e != cudaSuccess) return p->cuda_fail(e, "launch_agg");
        snprintf(p->stats.main_kernel_name, sizeof p->stats.main_kernel_name, "%s", agg_kernel_name(sel.kernel));
        p->stats.kernel_launches++;
    }
    return BKGPU_OK;
}

int bind_columns(bkgpu_plan* p, const std::vector<ColRef>& want, const bkgpu_column* cols, int ncols, int64_t nrows,
                 std::vector<const bkgpu_column*>& bound) {
    bound.assign(want.size(), nullptr);
    for (size_t i = 0; i < want.size(); i++) {
        for (int k = 0; k < ncols; k++) if (cols[k].tuple_id == want[i].tuple_id && cols[k].slot_id == want[i].slot_id) { bound[i] = &cols[k]; break; }
        if (!bound[i]) return p->fail(BKGPU_EINVAL, "batch lacks column %d_%d", want[i].tuple_id, want[i].slot_id);
        if (bound[i]->length != nrows) return p->fail(BKGPU_EINVAL, "column %d_%d has length %lld, batch has %lld rows", want[i].tuple_id,
                                                      want[i].slot_id, (long long)bound[i]->length, (long long)nrows);
        if (nrows > 0 && !bound[i]->values) return p->fail(BKGPU_EINVAL, "column %d_%d has no values buffer", want[i].tuple_id, want[i].slot_id);
        if (prim_storage(bound[i]->prim_type) != prim_storage(want[i].prim))
            return p->fail(BKGPU_EINVAL, "column %d_%d arrives as type %d but the plan declares %d", want[i].tuple_id, want[i].slot_id,
                           bound[i]->prim_type, want[i].prim);
    }
    return BKGPU_OK;
}

static int ensure_stage(bkgpu_plan* p, const std::vector<ColRef>& want, size_t rows) {
    if (p->stage_rows >= rows && p->stage[0].size() == want.size()) return BKGPU_OK;
    for (int b = 0; b < 2; b++) {
        for (void* q : p->stage[b]) dev_free(p, q);
        for (void* q : p->stage_valid[b]) dev_free(p, q);
        p->stage[b].assign(want.size(), nullptr); p->stage_valid[b].assign(want.size(), nullptr);
        for (size_t i = 0; i < want.size(); i++) {
            int rc;
            if ((rc = dev_alloc(p, &p->stage[b][i], rows * (size_t)storage_bytes(prim_storage(want[i].prim))))) return rc;
            if ((rc = dev_alloc(p, &p->stage_valid[b][i], rows / 8 + 8))) return rc;
        }
    }
    p->stage_rows = rows;
    return BKGPU_OK;
}

// pinned bounce buffers for pageable input: one per staging buffer set and column
static int ensure_bounce(bkgpu_plan* p, const std::vector<ColRef>& want, size_t rows) {
    if (p->bounce_rows >= rows && p->bounce[0].size() >= want.size()) return BKGPU_OK;
    for (int b = 0; b < 2; b++) {
        for (uint8_t* q : p->bounce[b]) if (q) cudaFreeHost(q);
        p->bounce[b].assign(want.size(), nullptr);
        for (size_t i = 0; i < want.size(); i++) {
            const size_t bytes = rows * (size_t)storage_bytes(prim_storage(want[i].prim));
            if (cudaHostAlloc((void**)&p->bounce[b][i], bytes ? bytes : 8, cudaHostAllocDefault) != cudaSuccess) return p->fail(BKGPU_ENOMEM, "pinned bounce buffer of %zu bytes", bytes);
        }
        if (!p->bounce_done[b]) CK(p, cudaEventCreateWithFlags(&p->bounce_done[b], cudaEventDisableTiming));
        p->bounce_busy[b] = false;
    }
    p->bounce_rows = rows;
    return BKGPU_OK;
}

// ---- host-side copy workers: pageable input (what an Arrow RecordBatch of RocksdbVectorizedReader hands over) is copied into
// pinned bounce buffers by several threads — cudaMemcpyAsync from pageable memory goes through the driver's single staging buffer
// at a fraction of the link rate ----
namespace bk { void stream_copy(void* dst, const void* src, size_t bytes); }   // hostcopy.cpp
namespace {
class CopyPool {
  public:
    explicit CopyPool(int n) { for (int i = 0; i < n; i++) th_.emplace_back([this] { run(); }); }
    ~CopyPool() { { std::lock_guard<std::mutex> g(mu_); stop_ = true; } cv_.notify_all(); for (auto& t : th_) t.join(); }
    int size() const { return (int)th_.size(); }
    // runs fn(0) .. fn(n - 1) on the workers and the caller; returns when all are done
    void parallel(int n, const std::function<void(int)>& fn) {
        if (n <= 0) return;
        {
            std::lock_guard<std::mutex> g(mu_);
            fn_ = &fn; next_ = 0; total_ = n; done_ = 0; gen_++;
        }
        cv_.notify_all();
        work();
        std::unique_lock<std::mutex> g(mu_);
        done_cv_.wait(g, [this] { return done_ == total_; });
        fn_ = nullptr;
    }
  private:
    void work() {
        for (;;) {
            int i;
            const std::function<void(int)>* f;
            { std::lock_guard<std::mutex> g(mu_); if (!fn_ || next_ >= total_) return; i = next_++; f = fn_; }
            (*f)(i);
            { std::lock_guard<std::mutex> g(mu_); ++done_; if (done_ == total_) done_cv_.notify_all(); }
        }
    }
    void run() {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> g(mu_);
                cv_.wait(g, [&] { return stop_ || gen_ != seen; });
                if (stop_) return;
                seen = gen_;
            }
            work();
        }
    }
    std::vector<std::thread> th_;
    std::mutex mu_; std::condition_variable cv_, done_cv_;
    const std::function<void(int)>* fn_ = nullptr;
    int next_ = 0, total_ = 0, done_ = 0; uint64_t gen_ = 0; bool stop_ = false;
};
// CPUs this process may actually use: online CPUs, its affinity mask and its cgroup CPU quota (a container with a 16-CPU quota on a 128-CPU box
// gets throttled for the rest of the scheduling period once its threads have burnt the quota — spinning or oversized pools make the copy SLOWER there)
int cpu_budget() {
    int n = (int)std::thread::hardware_concurrency();
    cpu_set_t set; CPU_ZERO(&set);
    if (sched_getaffinity(0, sizeof set, &set) == 0) { const int a = CPU_COUNT(&set); if (a > 0 && a < n) n = a; }
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {   // cgroup v2: "<quota|max> <period>"
        char q[32]; long long period = 0;
        if (fscanf(f, "%31s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) { const long long c = atoll(q) / period; if (c > 0 && c < n) n = (int)c; }
        fclose(f);
    } else if (FILE* g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {   // cgroup v1
        long long quota = -1, period = 100000;
        if (fscanf(g, "%lld", &quota) != 1) quota = -1;
        fclose(g);
        if (FILE* h = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) { if (fscanf(h, "%lld", &period) != 1) period = 100000; fclose(h); }
        if (quota > 0 && period > 0 && quota / period > 0 && quota / period < n) n = (int)(quota / period);
    }
    return n > 0 ? n : 1;
}
CopyPool& copy_pool() {
    static CopyPool pool([] {
        if (const char* e = getenv("BKGPU_COPY_THREADS")) { const int v = atoi(e); if (v > 0) return std::min(v, 64) - 1; }
        return std::max(1, std::min(23, cpu_budget() * 3 / 4 - 1));   // workers + the pushing thread = 3/4 of the CPU budget
                                                                       // (12 threads 0.895 of the pinned rate; 8: 0.82, 16: 0.85, 24: 0.81), 24 threads on an unconstrained host
    }());
    return pool;
}
bool is_pageable(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}
}  // namespace

// feed a batch: device-resident columns go straight to the kernels; host columns stream through
// two sets of device staging buffers (H2D of chunk i+1 overlaps the kernel on chunk i)
int feed(bkgpu_plan* p, const std::vector<ColRef>& want, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device, BatchFn fn) {
    std::vector<const bkgpu_column*> bound;
    int rc = bind_columns(p, want, cols, ncols, nrows, bound);
    if (rc) return rc;
    std::vector<DevCol> dc(std::max<size_t>(want.size(), 1));
    if (on_device) {
        bool vec_ok = true;
        for (size_t i = 0; i < want.size(); i++) {
            dc[i].values = bound[i]->values; dc[i].validity = bound[i]->validity;
            dc[i].stype = prim_storage(want[i].prim); dc[i].prim = want[i].prim;
            if (((uintptr_t)dc[i].values & 31) != 0) vec_ok = false;
        }
        return fn(p, dc.data(), nrows, 0, vec_ok);
    }
    bool pageable = false;
    for (size_t i = 0; i < want.size(); i++) pageable = pageable || is_pageable(bound[i]->values);
    // (pageable input adds a CPU copy stage of about the link's speed in front of the H2D copy: smaller chunks keep the fill / drain
    //  of that three-stage pipeline at ~2 % of the batch instead of ~8 %)
    int64_t chunk_cap = pageable ? std::min<int64_t>(p->chunk_rows, (int64_t)2 << 20) : p->chunk_rows;
    for (const ColRef& w : want)   // (a 16400-byte HLL sketch column: staging chunks of at most 256 MB per buffer, a multiple of 8 rows)
        if (prim_storage(w.prim) == ST_HLL) chunk_cap = std::min<int64_t>(chunk_cap, ((int64_t)256 << 20) / HLL_RAW_BYTES & ~7ll);
    const int64_t chunk = std::min<int64_t>(chunk_cap, std::max<int64_t>((nrows + 7) & ~7ll, 8));
    if ((rc = ensure_stage(p, want, (size_t)chunk))) return rc;
    if (pageable && (rc = ensure_bounce(p, want, (size_t)chunk))) return rc;
    int buf = 0;
    cudaEvent_t last_ready = nullptr;
    for (int64_t off = 0; off < nrows; off += chunk, buf ^= 1) {
        if (p->cancelled.load()) return p->fail(BKGPU_ECANCELLED, "cancelled");
        const int64_t n = std::min(chunk, nrows - off);
        CK(p, cudaStreamWaitEvent(p->copy_stream, p->stage_free[buf], 0));
        if (pageable) {   // bounce: worker threads fill this buffer set's pinned copy of the chunk, the link then runs at the pinned rate
            if (p->bounce_busy[buf]) { CK(p, cudaEventSynchronize(p->bounce_done[buf])); p->bounce_busy[buf] = false; }
            struct Piece { uint8_t* dst; const uint8_t* src; size_t bytes; };
            std::vector<Piece> pieces;
            const size_t slice = (size_t)1 << 20;
            for (size_t i = 0; i < want.size(); i++) {
                const size_t eb = (size_t)storage_bytes(prim_storage(want[i].prim)), bytes = (size_t)n * eb;
                const uint8_t* src = (const uint8_t*)bound[i]->values + (size_t)off * eb;
                for (size_t o = 0; o < bytes; o += slice) pieces.push_back({p->bounce[buf][i] + o, src + o, std::min(slice, bytes - o)});
            }
            copy_pool().parallel((int)pieces.size(), [&](int k) {
                const Piece& pc = pieces[(size_t)k];
                stream_copy(pc.dst, pc.src, pc.bytes);
            });
        }
        for (size_t i = 0; i < want.size(); i++) {
            const int st = prim_storage(want[i].prim);
            const size_t eb = (size_t)storage_bytes(st);
            const void* hsrc = pageable ? (const void*)p->bounce[buf][i] : (const void*)((const uint8_t*)bound[i]->values + (size_t)off * eb);
            CK(p, cudaMemcpyAsync(p->stage[buf][i], hsrc, (size_t)n * eb, cudaMemcpyHostToDevice, p->copy_stream));
            p->stats.h2d_bytes += (int64_t)((size_t)n * eb);
            dc[i].values = p->stage[buf][i]; dc[i].stype = st; dc[i].prim = want[i].prim; dc[i].validity = nullptr;
            if (bound[i]->validity) {
                CK(p, cudaMemcpyAsync(p->stage_valid[buf][i], bound[i]->validity + off / 8, (size_t)(n + 7) / 8, cudaMemcpyHostToDevice, p->copy_stream));
                p->stats.h2d_bytes += (n + 7) / 8;
                dc[i].validity = (const uint8_t*)p->stage_valid[buf][i];
            }
        }
        CK(p, cudaEventRecord(p->stage_ready[buf], p->copy_stream));
        if (pageable) { CK(p, cudaEventRecord(p->bounce_done[buf], p->copy_stream)); p->bounce_busy[buf] = true; }
        CK(p, cudaStreamWaitEvent(p->stream, p->stage_ready[buf], 0));
        if ((rc = fn(p, dc.data(), n, off, true))) return rc;
        CK(p, cudaEventRecord(p->stage_free[buf], p->stream));
        last_ready = p->stage_ready[buf];
    }
    // the caller's host buffers are borrowed for the duration of the call only (bkgpu.h): the last host-to-device copy must have
    // read them before bkgpu_push returns (the kernels read the staging buffers, they may still be running)
    if (last_ready) CK(p, cudaEventSynchronize(last_ready));
    return BKGPU_OK;
}

static int agg_batch(bkgpu_plan* p, const DevCol* cols, int64_t nrows, int64_t, bool vec_ok) { return launch_agg_batch(p, p->c, cols, nrows, vec_ok); }
static int sort_batch(bkgpu_plan* p, const DevCol* cols, int64_t nrows, int64_t, bool) { return sort_push(p->sort, cols, nrows, &p->stats); }

void set_result(bkgpu_plan* p, std::vector<SortOutCol>& cols, int64_t rows, const OutCol* desc) {
    p->result.clear();
    for (size_t k = 0; k < cols.size(); k++) {
        SortOutCol& sc = cols[k];
        HostCol hc; hc.desc = desc ? desc[k] : OutCol{sc.tuple_id, sc.slot_id, sc.prim, 0}; hc.elem = sc.elem;
        hc.values = std::move(sc.values); hc.validity = std::move(sc.validity);
        p->result.push_back(std::move(hc));
    }
    p->result_rows = rows; p->result_pos = 0;
}

// MERGE_AGG of hll_add_agg over host memory: every non-NULL input value must be a RAW sketch, or the push fails (device-resident input is
// checked by the merge kernel itself, and the request then fails at bkgpu_finish)
static int hll_check_host_sketches(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows) {
    const AggPlan& ap = p->c.ap;
    for (int k = 0; k < ap.n_agg; k++) {
        if (ap.agg[k].kind != AG_HLL || ap.agg[k].arg_prim != BK_HLL) continue;
        const ColRef& w = p->c.cols[ap.agg[k].hll_col];
        for (int i = 0; i < ncols; i++) {
            if (cols[i].tuple_id != w.tuple_id || cols[i].slot_id != w.slot_id || !cols[i].values || cols[i].length != nrows) continue;   // (bind_columns reports those)
            for (int64_t r = 0; r < nrows; r++) {
                if (cols[i].validity && !((cols[i].validity[r >> 3] >> (r & 7)) & 1)) continue;
                const uint8_t* v = (const uint8_t*)cols[i].values + (size_t)r * HLL_RAW_BYTES;
                if (memcmp(v, "HYLL", 4) != 0 || v[4] != HLL_ENC_RAW)
                    return p->fail(BKGPU_EINVAL, "column %d_%d row %lld is not a RAW HLL sketch (\"HYLL\", encoding 255, 16400 bytes): MERGE_AGG of hll_add_agg "
                                   "merges RAW sketches only", w.tuple_id, w.slot_id, (long long)r);
            }
        }
    }
    return BKGPU_OK;
}

static int bkgpu_push_impl(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device);
extern "C" int bkgpu_push(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    const double t0 = HostClock::now();
    const int rc = bkgpu_push_impl(p, cols, ncols, nrows, on_device);
    if (p) p->hclk.push += HostClock::now() - t0;
    return rc;
}
static int bkgpu_push_impl(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    if (!p) return thread_fail(BKGPU_EINVAL, "bkgpu_push: NULL plan");
    if (p->state != S_OPEN) return p->fail(BKGPU_ESTATE, "bkgpu_push needs an open, unfinished plan");
    if (p->cancelled.load()) return p->fail(BKGPU_ECANCELLED, "cancelled");
    if (nrows < 0 || ncols < 0 || (ncols > 0 && !cols)) return p->fail(BKGPU_EINVAL, "bkgpu_push: bad arguments");
    CK(p, cudaSetDevice(p->device));
    p->stats.rows_scanned += nrows;
    if (nrows == 0) return BKGPU_OK;
    switch (p->c.kind) {
        case PK_AGG: {
            int rc = on_device ? BKGPU_OK : hll_check_host_sketches(p, cols, ncols, nrows);
            if (rc) return rc;
            rc = feed(p, p->c.cols, cols, ncols, nrows, on_device, agg_batch);
            if (rc) return rc;
            // learn the cardinality for later batches' table size (no sync: a stale value only costs speed); a launch that extracted its
            // result has already left the count in h_fused
            if (p->c.ap.n_keyw > 0 && p->smem_cap_log2 < 0 && p->h_pinned && !p->fused_last)
                CK(p, cudaMemcpyAsync(p->h_pinned, p->gt.n_groups, 4, cudaMemcpyDeviceToHost, p->stream));
            return BKGPU_OK;
        }
        case PK_JOIN_AGG: case PK_JOIN: case PK_STAR_AGG: return join_push(p, cols, ncols, nrows, on_device);
        case PK_SORT: case PK_FILTER: case PK_WINDOW: return feed(p, p->c.cols, cols, ncols, nrows, on_device, sort_batch);
        default: return p->fail(BKGPU_EUNSUPPORTED, "plan kind %d has no push path yet", p->c.kind);
    }
}


// groups per rank in the exchanged partial state: never more than the group table can hold (every rank runs the same plan with
// the same options, so all ranks agree on it) — a 2^14-slot table ships 0.8 MB per rank instead of the 3 MB of the default cap
static uint32_t eff_pcap(const bkgpu_plan* p) {
    const int64_t table = p->c.ap.n_keyw == 0 ? 1 : (int64_t)1 << p->group_cap_log2;
    return (uint32_t)std::min<int64_t>(p->partial_cap, table);
}

// the collective step of bkgpu_finish: regions -> one set per GPU, the per-GPU partial tables meet once and are folded by K3.
// Default: compact rows, one ncclAllGather of 1 + bound x (key + lane words) per rank — `bound` = the largest group count any rank
// held in earlier runs of this plan (2048 on the first run); the merge reports the true maximum and the exchange is repeated once
// with a larger bound when it did not fit.  Option repartition: all-to-all by key owner.
static int agg_collective(bkgpu_plan* p, bool* rows_mode) {
    const AggPlan& ap = p->c.ap;
    GroupTable& gt = p->gt;
    *rows_mode = false;
    const uint32_t pcap = eff_pcap(p);
    int rc;
    const bool repart = p->repartition && ap.n_keyw > 0;   // (a scalar aggregate has one group: nothing to partition)
    EventPair* ep = timer_begin(p, p->timed_coll, 0);
    if (!repart) {
        *rows_mode = true;
        if (p->rank < 0 && nccl_comm_rank(p->nccl_comm, &p->rank) != 0) return p->fail(BKGPU_ENCCL, "ncclCommUserRank: %s", nccl_last_error());
        uint32_t bound = p->merge_bound ? p->merge_bound : 2048u;
        if (ap.n_keyw == 0) bound = 1;
        bound = std::min<uint32_t>(bound, pcap);
        const size_t rw = (size_t)(ap.n_keyw + ap.n_lanes + ap.n_hll * HLL_ROW_WORDS);
        const size_t words = 1 + rw * bound;
        if ((rc = ensure_buf(p, (void**)&p->d_partial, &p->d_partial_cap, words * 8))) return rc;
        if ((rc = ensure_buf(p, (void**)&p->d_gather, &p->d_gather_cap, words * 8 * (size_t)p->nranks))) return rc;
        CK(p, launch_partial_export_rows(gt, ap, p->d_partial, bound, p->stream));
        if (nccl_all_gather(p->nccl_comm, p->d_partial, p->d_gather, words, p->stream) != 0) return p->fail(BKGPU_ENCCL, "ncclAllGather: %s", nccl_last_error());
        CK(p, launch_partial_merge_rows(gt, ap, p->d_gather, words, bound, p->nranks, p->rank, p->d_cursor + 1, p->stream));
        p->merge_bound_used = bound;
        p->stats.kernel_launches += 2;
        timer_end(p, ep);
        return BKGPU_OK;
    }
    // hash repartition: every rank keeps only the groups it owns — an all-to-all of per-owner segments instead of the
    // all-gather; the merged table (and the result) of a rank is its partition, the union over ranks is the answer
    const size_t words = 1 + (size_t)(ap.n_keyw + ap.n_lanes) * pcap;
    if ((rc = ensure_buf(p, (void**)&p->d_partial, &p->d_partial_cap, words * 8 * (size_t)p->nranks))) return rc;
    if ((rc = ensure_buf(p, (void**)&p->d_gather, &p->d_gather_cap, words * 8 * (size_t)p->nranks))) return rc;
    if (!p->d_part_cursors && (rc = dev_alloc(p, (void**)&p->d_part_cursors, 4 * (size_t)p->nranks))) return rc;
    CK(p, launch_partial_export_parts(gt, ap, p->d_partial, words, pcap, p->d_part_cursors, p->nranks, p->stream));
    if (nccl_all_to_all(p->nccl_comm, p->d_partial, p->d_gather, words, p->nranks, p->stream) != 0) return p->fail(BKGPU_ENCCL, "all-to-all: %s", nccl_last_error());
    CK(p, launch_table_init(gt, ap, p->stream, 1));   // (keeps the overflow flag an export beyond partial_capacity raised)
    CK(p, launch_partial_merge(gt, ap, p->d_gather, words, pcap, p->nranks, p->stream));
    timer_end(p, ep);
    p->stats.kernel_launches += 4;
    return BKGPU_OK;
}

// [LIMIT ->] [SORT ->] [HAVING ->] above the aggregate: the extracted rows (still on the device) become typed columns and run through
// the post fragment's sort / filter kernels; only the final rows travel to the host
static int agg_post(bkgpu_plan* p, uint32_t n_out, uint32_t out_cap) {
    const Compiled& pc = *p->c.post;
    const size_t nc = pc.cols.size();
    int rc;
    for (size_t c = 0; c < nc; c++)
        if ((rc = store_reserve(p, p->post, c, std::max<int64_t>(n_out, 1), std::max<int64_t>(n_out, 2048), true))) return rc;
    PostCols pcs; memset(&pcs, 0, sizeof pcs);
    pcs.n = (int)nc;
    int img = 0;
    for (size_t c = 0; c < nc; c++) {   // (post columns = the aggregate's output columns, in order: plan.cpp::lower_post)
        pcs.img[c] = img; pcs.stype[c] = prim_storage(pc.cols[c].prim); pcs.values[c] = p->post.cols[c].vals; pcs.null_bytes[c] = p->post.cols[c].nulls;
        img += p->c.out_cols[c].kind == 1 ? 2 : 1;
    }
    CK(p, launch_images_to_columns(p->d_outv, p->d_outn, out_cap, n_out, pcs, p->stream));
    std::vector<DevCol> dc(std::max<size_t>(nc, 1));
    for (size_t c = 0; c < nc; c++)
        if ((rc = store_pack(p, p->post, c, n_out, 16, nullptr, &dc[c]))) return rc;
    p->stats.kernel_launches += 1 + (int64_t)nc;
    sort_reset(p->post_sort);
    bkgpu_stats scratch{};   // (the post fragment's kernels are not the request's "main kernel")
    if (n_out && (rc = sort_push(p->post_sort, dc.data(), n_out, &scratch))) return rc;
    std::vector<SortOutCol> cols; int64_t rows = 0;
    if ((rc = sort_finish(p->post_sort, nullptr, 1, &scratch, cols, &rows))) return rc;
    p->stats.kernel_launches += scratch.kernel_launches;
    set_result(p, cols, rows, p->c.out_cols.data());
    return BKGPU_OK;
}

// the one wait of a request.  With several ranks on a host whose CPU budget is small (8 ranks under a 16-CPU cgroup quota: two CPUs per
// rank for the python thread, NCCL's proxy thread and this wait) a spinning wait burns the quota the other ranks' launches need:
// there the thread sleeps on a blocking-sync event instead (option blocking_sync: -1 auto, 0 spin, 1 sleep)
static int agg_wait(bkgpu_plan* p) {
    const double t0 = HostClock::now();
    if (p->blocking_wait) {
        if (!p->wait_event) CK(p, cudaEventCreateWithFlags(&p->wait_event, cudaEventBlockingSync | cudaEventDisableTiming));
        CK(p, cudaEventRecord(p->wait_event, p->stream));
        CK(p, cudaEventSynchronize(p->wait_event));
    } else CK(p, cudaStreamSynchronize(p->stream));
    p->hclk.extract_wait += HostClock::now() - t0;
    return BKGPU_OK;
}

// what the counter block of a finished request tells the plan: rows that passed, FX's exact-path count, the groups it holds
static int agg_take_counters(bkgpu_plan* p, const uint32_t* ctr) {
    memcpy(&p->rows_passed_host, ctr + 4, 8);
    // FX: values beyond the sampled scale are added exactly, one global atomic each; a plan whose double columns keep producing many of them
    // (a column spanning dozens of binades, outliers dominating the sample) goes back to the CAS kernel for its later launches
    if (ctr[GT_FX_EXACT] > 4096 && (uint64_t)ctr[GT_FX_EXACT] * 64 > (uint64_t)std::max<int64_t>(p->rows_passed_host, 1)) p->fx_off = 1;
    if (ctr[1]) return p->fail(BKGPU_ETOOBIG, "group table overflow (capacity 2^%d slots / partial_capacity %lld): raise group_capacity_log2",
                               (int)p->gt.cap_log2, (long long)p->partial_cap);
    if (ctr[0] > p->known_groups) p->known_groups = ctr[0];
    p->finish_groups = ctr[0];
    return BKGPU_OK;
}

// a BITMAP column (bkgpu.h): one bitmap per row, each the device's bytes for (slot, rb_idx), or the 8-byte empty bitmap
// ("3a300000 00000000": the reference's initialize gives every group an empty bitmap, so a group whose values were all NULL returns it)
static void rb_column(bkgpu_plan* p, HostCol& hc, const uint64_t* slot, int64_t rows, int rb_idx) {
    static const uint8_t empty[8] = {0x3a, 0x30, 0, 0, 0, 0, 0, 0};
    std::vector<int64_t> b((size_t)rows);   // each row's bitmap in the directory, -1 = none
    int64_t total = 0;
    for (int64_t r = 0; r < rows; r++) {
        const uint32_t id = (uint32_t)(slot[r] << 2) | (uint32_t)rb_idx;
        const auto it = std::lower_bound(p->rb.bid.begin(), p->rb.bid.end(), id);
        b[r] = it != p->rb.bid.end() && *it == id ? (int64_t)(it - p->rb.bid.begin()) : -1;
        total += b[r] < 0 ? 8 : (int64_t)(p->rb.off[b[r] + 1] - p->rb.off[b[r]]);
    }
    std::vector<uint8_t>& col = p->rb.col[rb_idx];
    col.resize(((size_t)rows + 1) * 8 + (size_t)total);
    int64_t* offs = (int64_t*)col.data();
    uint8_t* d = col.data() + ((size_t)rows + 1) * 8;
    offs[0] = 0;
    for (int64_t r = 0; r < rows; r++) {
        const size_t len = b[r] < 0 ? 8 : (size_t)(p->rb.off[b[r] + 1] - p->rb.off[b[r]]);
        memcpy(d + offs[r], b[r] < 0 ? empty : p->rb.bytes + p->rb.off[b[r]], len);
        offs[r + 1] = offs[r] + (int64_t)len;
    }
    hc.elem = -1;
    hc.varlen = &col;
}

// typed host columns from `n_out` extracted rows (images + null bytes, column-major with stride `stride`), after OFFSET / LIMIT
static void agg_result(bkgpu_plan* p, const uint64_t* hv, const uint8_t* hn, size_t stride, uint32_t n_out) {
    const int64_t rows = n_out;
    const int64_t skip = p->c.offset > 0 ? std::min<int64_t>(p->c.offset, rows) : 0;
    int64_t lim = p->c.agg_limit;   // AggNode::get_next stops at its limit (agg_node.cpp:555)
    if (p->c.limit >= 0 && (lim < 0 || p->c.limit < lim)) lim = p->c.limit;
    int64_t keep = rows - skip;
    if (lim >= 0 && keep > lim) keep = lim;
    p->result.clear();
    int img = 0, rb_idx = 0;
    for (const OutCol& oc : p->c.out_cols) {
        HostCol hc; hc.desc = oc;
        const uint64_t* v = hv + (size_t)img * stride + skip;
        const uint8_t* nb = hn + (size_t)img * stride + skip;
        if (oc.kind == 3) {   // rb_build_agg: the group's slot, whose bitmap the device build serialized (a group without a value: the empty one)
            rb_column(p, hc, v, keep, rb_idx++);
            img++;
            p->result.push_back(std::move(hc));
            continue;
        }
        hc.elem = oc.kind == 1 ? 16 : oc.kind == 2 ? HLL_RAW_BYTES : storage_bytes(prim_storage(oc.prim));
        hc.values.assign((size_t)std::max<int64_t>(keep, 1) * (size_t)hc.elem, 0);
        // (a NULL's image is 0, which is also what a NULL row's value bytes hold)
        uint8_t* d = hc.values.data();
        if (oc.kind == 1) {
            const uint64_t* v2 = hv + (size_t)(img + 1) * stride + skip;
            for (int64_t r = 0; r < keep; r++) { memcpy(d + (size_t)r * 16, v + r, 8); memcpy(d + (size_t)r * 16 + 8, v2 + r, 8); }
        } else if (oc.kind == 2) {
            // hll_row_init's RAW sketch (hll_common.cpp:834-842): "HYLL", encoding HLL_RAW, then the registers.  hll_row_add invalidates the
            // cached cardinality (bit 7 of header byte 15) whenever a register grows, which the first value always does: a group that
            // received a value has the bit set, a group without one (every argument NULL) is the empty sketch with the byte 0
            for (int64_t r = 0; r < keep; r++) {
                uint8_t* o = d + (size_t)r * HLL_RAW_BYTES;
                memcpy(o, "HYLL", 4); o[4] = HLL_ENC_RAW;
                if (v[r]) { o[15] = 0x80; memcpy(o + HLL_HDR_BYTES, p->hll_host.data() + (size_t)(v[r] - 1) * HLL_REGISTERS, HLL_REGISTERS); }
            }
        } else switch (prim_storage(oc.prim)) {
            case ST_I32: for (int64_t r = 0; r < keep; r++) { const int32_t x = (int32_t)(int64_t)v[r]; memcpy(d + (size_t)r * 4, &x, 4); } break;
            case ST_U32: for (int64_t r = 0; r < keep; r++) { const uint32_t x = (uint32_t)v[r]; memcpy(d + (size_t)r * 4, &x, 4); } break;
            case ST_F32: for (int64_t r = 0; r < keep; r++) { double x; memcpy(&x, v + r, 8); const float f = (float)x; memcpy(d + (size_t)r * 4, &f, 4); } break;
            case ST_U8: for (int64_t r = 0; r < keep; r++) d[r] = v[r] ? 1 : 0; break;
            default:
                if (hc.elem == 8) { if (keep > 0) memcpy(d, v, (size_t)keep * 8); }
                else for (int64_t r = 0; r < keep; r++) memcpy(d + (size_t)r * hc.elem, v + r, 8);
                break;
        }
        if (keep > 0 && memchr(nb, 1, (size_t)keep)) {
            hc.validity.assign((size_t)(keep + 7) / 8 + 1, 0xFF);
            for (int64_t r = 0; r < keep; r++) if (nb[r]) { hc.validity[(size_t)r >> 3] &= (uint8_t)~(1u << (r & 7)); if (oc.kind == 0) memset(d + (size_t)r * hc.elem, 0, (size_t)hc.elem); }
        }
        img += oc.kind == 1 ? 2 : 1;
        p->result.push_back(std::move(hc));
    }
    p->result_rows = keep; p->result_pos = 0;
}

// hll_add_agg: the arena's claimed blocks to the host (the extracted rows reference them), after the request's last kernel.  A claim
// that found the arena full fails the request: a sketch that lost values would be wrong, not approximate
static int hll_fetch(bkgpu_plan* p) {
    if (!p->c.ap.n_hll) return BKGPU_OK;
    uint32_t ctr[3] = {0, 0, 0};
    CK(p, cudaMemcpyAsync(ctr, p->gt.hll_ctr, 12, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    if (ctr[2]) return p->fail(BKGPU_EINVAL, "MERGE_AGG of hll_add_agg: an input value is not a RAW HLL sketch (\"HYLL\", encoding 255, 16400 bytes)");
    if (ctr[1] || ctr[0] > p->gt.hll_cap)
        return p->fail(BKGPU_ETOOBIG, "hll_add_agg: more than %u sketches (groups x hll_add_agg aggregates with a value): raise hll_group_capacity",
                       p->gt.hll_cap);
    p->hll_host.resize((size_t)ctr[0] * HLL_REGISTERS);
    if (ctr[0]) CK(p, cudaMemcpy(p->hll_host.data(), p->gt.hll_regs, (size_t)ctr[0] * HLL_REGISTERS, cudaMemcpyDeviceToHost));
    p->stats.d2h_bytes += (int64_t)p->hll_host.size() + 8;
    return BKGPU_OK;
}

static int agg_finish(bkgpu_plan* p) {
    const AggPlan& ap = p->c.ap;
    GroupTable& gt = p->gt;
    uint32_t host_counts[2] = {0, 0};
    uint64_t* finish_hv = nullptr; uint8_t* finish_hn = nullptr; uint32_t finish_n_out = 0, finish_out_cap = 0;
    const bool multi = p->nccl_comm && p->nranks > 1;
    bool rows_mode = false;
    const int n_img = agg_n_img(ap);
    int rc;
    // the request ended with a launch that extracted its own result into mapped host memory: one wait, nothing else on the device
    if (p->fused_last && !multi && !p->c.post) {
        if ((rc = agg_wait(p))) return rc;
        const uint32_t* ctr = (const uint32_t*)p->h_fused;
        if ((rc = agg_take_counters(p, ctr))) return rc;
        const uint32_t n = ctr[0];
        if (n <= p->fused_cap) {
            p->stats.d2h_bytes += (int64_t)(32 + (size_t)n * (size_t)n_img * 9);
            const uint64_t* hv = (const uint64_t*)(p->h_fused + 32);
            agg_result(p, hv, (const uint8_t*)(hv + (size_t)n * (size_t)n_img), n, n);
            return BKGPU_OK;
        }
        // more groups than the buffer holds: the table is read back below (the next launch's buffer is sized for them)
    }
  for (int mtry = 0; mtry < 3; mtry++) {   // (a second trip only when some rank held more groups than the exchange was sized for)
    { const double t0 = HostClock::now(); if (multi && (rc = agg_collective(p, &rows_mode))) return rc; p->hclk.collective += HostClock::now() - t0; }
    uint32_t n_out = 0, out_cap = 0, merge_max = 0;
    uint64_t* hv = nullptr; uint8_t* hn = nullptr;
    bool redo_merge = false;
    for (int attempt = 0; attempt < 2; attempt++) {
        // speculative extraction into the buffers kept from earlier runs: counts, cursor and rows come back
        // in ONE synchronisation; only a result larger than the buffers costs a second round
        uint32_t want = std::max<uint32_t>(std::max<uint32_t>(p->known_groups, 1), attempt ? std::max<uint32_t>(host_counts[0], 1) : 1);
        if (ap.n_keyw == 0) want = 1;
        if (p->out_cap_alloc < want) {
            dev_free(p, p->d_outv); p->d_outv = nullptr; p->d_outn = nullptr;
            size_t cap = std::max<size_t>(want, 2048);
            if ((rc = dev_alloc(p, (void**)&p->d_outv, cap * 9 * (size_t)n_img + 64))) return rc;   // values, then the null bytes: ONE copy brings both back
            p->d_outn = (uint8_t*)(p->d_outv + cap * (size_t)n_img);
            p->out_cap_alloc = cap;
        }
        out_cap = (uint32_t)p->out_cap_alloc;
        CK(p, launch_extract(gt, ap, p->d_outv, p->d_outn, out_cap, p->d_cursor, p->c.emit_default ? 1 : 0, p->stream));
        p->stats.kernel_launches++;
        const size_t n_words = (size_t)out_cap * (size_t)n_img;
        if (p->h_out_cap < n_words) {   // pinned: the four copies below are truly asynchronous and land in one synchronisation
            if (p->h_outv) cudaFreeHost(p->h_outv);
            p->h_outv = nullptr; p->h_outn = nullptr; p->h_out_cap = 0;
            CK(p, cudaHostAlloc((void**)&p->h_outv, n_words * 9 + 64, cudaHostAllocDefault));
            p->h_out_cap = n_words;
        }
        hv = p->h_outv; hn = p->h_outn = (uint8_t*)(p->h_outv + n_words);
        // two copies, one synchronisation: the 32-byte counter block (groups, overflow, rows extracted, merge info, rows passed) and
        // the extracted rows (values + null bytes, contiguous on both sides)
        uint32_t local_ctr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        uint32_t* hc3 = p->h_pinned ? p->h_pinned + 8 : local_ctr;   // [8] groups [9] overflow [10] rows extracted [11] merge info [12..13] rows passed
        CK(p, cudaMemcpyAsync(hc3, gt.n_groups, 32, cudaMemcpyDeviceToHost, p->stream));
        if ((const uint8_t*)p->d_outn == (const uint8_t*)(p->d_outv + n_words)) CK(p, cudaMemcpyAsync(hv, p->d_outv, n_words * 9, cudaMemcpyDeviceToHost, p->stream));
        else {
            CK(p, cudaMemcpyAsync(hv, p->d_outv, n_words * 8, cudaMemcpyDeviceToHost, p->stream));
            CK(p, cudaMemcpyAsync(hn, p->d_outn, n_words, cudaMemcpyDeviceToHost, p->stream));
        }
        if ((rc = agg_wait(p))) return rc;
        host_counts[0] = hc3[0]; host_counts[1] = hc3[1]; n_out = hc3[2]; merge_max = hc3[3];
        if (rows_mode) {
            const uint32_t mx = merge_max;
            if (mx > p->merge_bound_used) {   // nothing was merged (k_partial_merge_rows): exchange again, sized for what the ranks really hold
                if (mx > eff_pcap(p)) return p->fail(BKGPU_ETOOBIG, "a rank holds %u groups, more than partial_capacity %lld: raise partial_capacity", mx, (long long)p->partial_cap);
                p->merge_bound = (mx + 63u) & ~63u;
                redo_merge = true;
                break;
            }
            const uint32_t learned = (std::max<uint32_t>(mx, 1u) + 63u) & ~63u;
            if (learned > p->merge_bound) p->merge_bound = learned;
        }
        p->stats.d2h_bytes += (int64_t)(n_words * 9 + 12);
        if ((rc = agg_take_counters(p, hc3))) return rc;
        if (n_out <= out_cap) break;   // everything fitted
    }
    if (!redo_merge) { finish_hv = hv; finish_hn = hn; finish_n_out = n_out; finish_out_cap = out_cap; break; }
    if (mtry == 2) return p->fail(BKGPU_ENCCL, "partial-state exchange did not converge");
  }
    uint32_t n_out = finish_n_out, out_cap = finish_out_cap;
    if (n_out > out_cap) n_out = out_cap;
    if ((rc = hll_fetch(p))) return rc;
    if (p->c.n_rb && (rc = rb_build(p))) return rc;
    if (p->c.post) return agg_post(p, n_out, out_cap);
    agg_result(p, finish_hv, finish_hn, out_cap, n_out);
    return BKGPU_OK;
}

static void resolve_timers(bkgpu_plan* p) {
    for (auto& ep : p->timed) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ep.a, ep.b) == cudaSuccess) { p->stats.main_kernel_ms += ms; p->stats.main_kernel_launches++; p->stats.main_kernel_bytes += ep.bytes; }
        p->event_pool.push_back(ep.a); p->event_pool.push_back(ep.b);
    }
    p->timed.clear();
    for (auto& ep : p->timed_coll) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ep.a, ep.b) == cudaSuccess) p->stats.collective_ms += ms;
        p->event_pool.push_back(ep.a); p->event_pool.push_back(ep.b);
    }
    p->timed_coll.clear();
}

static int bkgpu_finish_impl(bkgpu_plan* p);
extern "C" int bkgpu_finish(bkgpu_plan* p) {
    const double t0 = HostClock::now();
    const int rc = bkgpu_finish_impl(p);
    if (p) { p->hclk.finish += HostClock::now() - t0; p->hclk.n++; }
    return rc;
}
static int bkgpu_finish_impl(bkgpu_plan* p) {
    if (!p) return thread_fail(BKGPU_EINVAL, "bkgpu_finish: NULL plan");
    if (p->state != S_OPEN) return p->fail(BKGPU_ESTATE, "bkgpu_finish needs an open plan");
    if (p->cancelled.load()) return p->fail(BKGPU_ECANCELLED, "cancelled");
    CK(p, cudaSetDevice(p->device));
    int rc = BKGPU_OK;
    switch (p->c.kind) {
        case PK_AGG: case PK_JOIN_AGG: case PK_STAR_AGG: {
            if (p->c.kind == PK_JOIN_AGG && (rc = join_tail(p))) break;
            rc = agg_finish(p);
            if (!rc) {
                p->stats.rows_filtered = p->stats.rows_scanned - (int64_t)p->rows_passed_host;   // (came back with the counter block)
            }
        } break;
        case PK_JOIN: {   // the outer join's preserved rows, then the sink fragment's result
            std::vector<SortOutCol> cols; int64_t rows = 0;
            if ((rc = join_tail(p)) || (rc = sort_finish(p->post_sort, nullptr, 1, &p->stats, cols, &rows))) break;
            set_result(p, cols, rows, p->c.out_cols.data());
            p->stats.rows_filtered = 0;
        } break;
        case PK_SORT: case PK_FILTER: {
            std::vector<SortOutCol> cols; int64_t rows = 0;
            if ((rc = sort_finish(p->sort, p->nccl_comm, p->nranks, &p->stats, cols, &rows))) break;
            set_result(p, cols, rows, nullptr);
        } break;
        case PK_WINDOW: {   // the retained rows through the window stages (window.cu), then the query's ORDER BY when there is one
            if (p->nccl_comm && p->nranks > 1) { rc = p->fail(BKGPU_EUNSUPPORTED, "a window fragment runs on one GPU: multi-GPU merge is implemented for ORDER BY ... LIMIT (top-k) and aggregates"); break; }
            std::vector<SortOutCol> cols; int64_t rows = 0;
            if ((rc = window_finish(p, cols, &rows))) break;
            set_result(p, cols, rows, nullptr);
        } break;
        default: rc = p->fail(BKGPU_EUNSUPPORTED, "plan kind %d cannot finish", p->c.kind);
    }
    // (a finished aggregate without a post fragment has already waited for everything it queued: agg_wait)
    if (rc || !((p->c.kind == PK_AGG || p->c.kind == PK_JOIN_AGG || p->c.kind == PK_STAR_AGG) && !p->c.post)) cudaStreamSynchronize(p->stream);
    resolve_timers(p);
    if (rc) return rc;
    p->stats.rows_returned = p->result_rows;
    p->state = S_FINISHED;
    return BKGPU_OK;
}

extern "C" int bkgpu_get_next(bkgpu_plan* p, bkgpu_column* out_cols, int* ncols, int64_t* nrows, int* eos) {
    if (!p || !ncols || !nrows || !eos) return thread_fail(BKGPU_EINVAL, "bkgpu_get_next: NULL argument");
    if (p->state != S_FINISHED) return p->fail(BKGPU_ESTATE, "bkgpu_get_next before bkgpu_finish");
    if (p->cancelled.load()) { *eos = 1; *nrows = 0; *ncols = 0; return BKGPU_OK; }  // cancelled: eos, like the reference's operators
    const int have = (int)p->result.size();
    if (*ncols < have || (have > 0 && !out_cols)) return p->fail(BKGPU_EINVAL, "bkgpu_get_next: need room for %d columns", have);
    const int64_t n = std::min(p->batch_capacity, p->result_rows - p->result_pos);
    for (int i = 0; i < have; i++) {
        HostCol& hc = p->result[(size_t)i];
        bkgpu_column& o = out_cols[i];
        o.tuple_id = hc.desc.tuple_id; o.slot_id = hc.desc.slot_id; o.prim_type = hc.desc.prim; o.elem_size = hc.elem;
        if (hc.elem < 0) {   // variable-length values: this batch's n + 1 offsets (from 0), then its bytes
            const int64_t* all = (const int64_t*)hc.varlen->data();
            const uint8_t* bytes = hc.varlen->data() + ((size_t)p->result_rows + 1) * 8;
            if (p->result_pos == 0 && n == p->result_rows) o.values = hc.varlen->data();   // (the whole column in one batch: as it is)
            else {
                const int64_t b0 = all[p->result_pos], b1 = all[p->result_pos + n];
                hc.batch.resize(((size_t)n + 1) * 8 + (size_t)(b1 - b0));
                int64_t* offs = (int64_t*)hc.batch.data();
                for (int64_t r = 0; r <= n; r++) offs[r] = all[p->result_pos + r] - b0;
                if (b1 > b0) memcpy(hc.batch.data() + ((size_t)n + 1) * 8, bytes + b0, (size_t)(b1 - b0));
                o.values = hc.batch.data();
            }
        } else
        o.values = hc.values.data() + (size_t)p->result_pos * (size_t)hc.elem;
        o.length = n;
        o.validity = nullptr;
        if (!hc.validity.empty()) {
            if (p->result_pos == 0) o.validity = hc.validity.data();
            else {  // re-base the bitmap for a non-first batch (batch_capacity is normally a multiple of 8)
                if (p->result_pos % 8 == 0) o.validity = hc.validity.data() + p->result_pos / 8;
                else return p->fail(BKGPU_EINVAL, "batch_capacity must be a multiple of 8 when results hold NULLs");
            }
        }
    }
    *ncols = have; *nrows = n;
    p->result_pos += n;
    *eos = p->result_pos >= p->result_rows ? 1 : 0;
    return BKGPU_OK;
}

// Re-arm an executed plan for the next request of the same fragment (prepared-statement reuse): tables
// are cleared, allocations, streams and staging buffers are kept.
static int bkgpu_reset_impl(bkgpu_plan* p);
extern "C" int bkgpu_reset(bkgpu_plan* p) {
    const double t0 = HostClock::now();
    const int rc = bkgpu_reset_impl(p);
    if (p) p->hclk.reset += HostClock::now() - t0;
    return rc;
}
static int bkgpu_reset_impl(bkgpu_plan* p) {
    if (!p) return thread_fail(BKGPU_EINVAL, "bkgpu_reset: NULL plan");
    if (p->state != S_OPEN && p->state != S_FINISHED) return p->fail(BKGPU_ESTATE, "bkgpu_reset needs an opened plan");
    CK(p, cudaSetDevice(p->device));
    p->cancelled.store(0);
    if (p->c.kind == PK_AGG || p->c.kind == PK_JOIN_AGG || p->c.kind == PK_STAR_AGG) {
        // a finished run knows how many groups its table holds (the count came back with the result): clear those slots through the
        // occupied list instead of re-initialising the whole capacity (2^20 slots = 44 MB by default)
        if (p->state == S_FINISHED && p->finish_groups >= 0 && p->c.ap.n_keyw > 0) CK(p, launch_table_clear(p->gt, p->c.ap, (uint32_t)p->finish_groups, p->stream));
        else CK(p, launch_table_init(p->gt, p->c.ap, p->stream));
        p->finish_groups = -1;
        p->fused_last = false;
        if (p->rb.ctr) { CK(p, cudaMemsetAsync(p->rb.ctr, 0, 8, p->stream)); p->rb.hi = 0; }   // (rb_build_agg: the pair buffer is empty again)
        p->stats.kernel_launches++;
    }
    join_reset(p);
    if (p->sort) sort_reset(p->sort);
    if (p->c.kind == PK_JOIN && p->post_sort) sort_reset(p->post_sort);
    p->result.clear(); p->result_rows = 0; p->result_pos = 0;
    bkgpu_stats z{}; z.kernel_launches = p->stats.kernel_launches; p->stats = z;
    p->state = S_OPEN;
    return BKGPU_OK;
}

extern "C" void bkgpu_cancel(bkgpu_plan* p) { if (p) p->cancelled.store(1); }

extern "C" void bkgpu_close(bkgpu_plan* p) {
    if (!p) return;
    if (p->trace && p->hclk.n) {
        const double n = (double)p->hclk.n;
        fprintf(stderr, "[bkgpu trace dev %d] %lld requests: host ms per request  reset %.4f  push %.4f  finish %.4f (collective enqueue %.4f, wait for the result %.4f)\n",
                p->device, (long long)p->hclk.n, p->hclk.reset / n, p->hclk.push / n, p->hclk.finish / n, p->hclk.collective / n, p->hclk.extract_wait / n);
    }
    cudaSetDevice(p->device);
    if (p->stream) cudaStreamSynchronize(p->stream);
    if (p->copy_stream) cudaStreamSynchronize(p->copy_stream);
    resolve_timers(p);
    if (p->sort) sort_close(p->sort);
    if (p->post_sort) sort_close(p->post_sort);
    for (cudaEvent_t e : p->event_pool) cudaEventDestroy(e);
    for (auto& q : p->dev_allocs) if (!dev_cache().put(p->device, q.second, q.first)) cudaFree(q.first);   // (both streams were drained above)
    for (int i = 0; i < 2; i++) { if (p->stage_free[i]) cudaEventDestroy(p->stage_free[i]); if (p->stage_ready[i]) cudaEventDestroy(p->stage_ready[i]); }
    for (int i = 0; i < 2; i++) { for (uint8_t* q : p->bounce[i]) if (q) cudaFreeHost(q); if (p->bounce_done[i]) cudaEventDestroy(p->bounce_done[i]); }
    if (p->wait_event) cudaEventDestroy(p->wait_event);
    if (p->h_pinned) cudaFreeHost(p->h_pinned);
    if (p->h_outv) cudaFreeHost(p->h_outv);
    if (p->rb.bytes) cudaFreeHost(p->rb.bytes);
    if (p->h_fused && !mapped_cache().put(p->fused_bytes, p->h_fused)) cudaFreeHost(p->h_fused);   // (the stream was drained above)
    if (p->copy_stream) cudaStreamDestroy(p->copy_stream);
    if (p->own_stream && p->stream) cudaStreamDestroy(p->stream);
    delete p;
}

extern "C" int bkgpu_get_stats(bkgpu_plan* p, bkgpu_stats* out) {
    if (!p || !out) return thread_fail(BKGPU_EINVAL, "bkgpu_get_stats: NULL argument");
    *out = p->stats;
    return BKGPU_OK;
}

// ------------------------------------------------------------------ resident regions
// A region's columns can be registered once and stay in HBM across queries (the reference's analogue: its column store and parquet
// cache keep hot regions decoded in memory, include/column/file_manager.h:252-272): 180 GB hold ~7e9 rows of the C2 shape, and a query
// over a resident region moves no input over PCIe at all.  Keyed by (device, region id); re-registering an id replaces it.
namespace {
struct ResidentRegion { int64_t nrows = 0; size_t bytes = 0; std::vector<bkgpu_column> cols; std::vector<void*> allocs; };
std::mutex g_region_mu;
std::map<std::pair<int, int64_t>, ResidentRegion> g_regions;
void free_region(ResidentRegion& r) { for (void* q : r.allocs) cudaFree(q); r.allocs.clear(); r.cols.clear(); r.bytes = 0; }
}  // namespace

extern "C" int bkgpu_region_register(int device, int64_t region_id, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    if (!cols || ncols <= 0 || nrows < 0) return thread_fail(BKGPU_EINVAL, "bkgpu_region_register: bad arguments");
    if (cudaSetDevice(device) != cudaSuccess) return thread_fail(BKGPU_ENODEV, "cudaSetDevice failed");
    ResidentRegion r; r.nrows = nrows;
    cudaStream_t st = nullptr;
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) return thread_fail(BKGPU_ENODEV, "cudaStreamCreate failed");
    int rc = BKGPU_OK;
    for (int i = 0; i < ncols && rc == BKGPU_OK; i++) {
        const bkgpu_column& c = cols[i];
        const int stype = prim_storage(c.prim_type);
        if (stype < 0 || c.length != nrows || (nrows > 0 && !c.values)) { rc = thread_fail(BKGPU_EINVAL, "bkgpu_region_register: column %d_%d is malformed", c.tuple_id, c.slot_id); break; }
        const size_t vb = (size_t)nrows * (size_t)storage_bytes(stype), nb = c.validity ? (size_t)(nrows + 7) / 8 : 0;
        void *dv = nullptr, *dn = nullptr;
        if (cudaMalloc(&dv, vb + 64) != cudaSuccess) { rc = thread_fail(BKGPU_ENOMEM, "cudaMalloc of %zu bytes failed", vb); break; }
        r.allocs.push_back(dv);
        if (nb) { if (cudaMalloc(&dn, nb + 64) != cudaSuccess) { rc = thread_fail(BKGPU_ENOMEM, "cudaMalloc of %zu bytes failed", nb); break; } r.allocs.push_back(dn); }
        const cudaMemcpyKind k = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        if (vb && cudaMemcpyAsync(dv, c.values, vb, k, st) != cudaSuccess) { rc = thread_fail(BKGPU_ENODEV, "copy of column %d_%d failed", c.tuple_id, c.slot_id); break; }
        if (nb && cudaMemcpyAsync(dn, c.validity, nb, k, st) != cudaSuccess) { rc = thread_fail(BKGPU_ENODEV, "copy of column %d_%d failed", c.tuple_id, c.slot_id); break; }
        bkgpu_column d = c; d.values = dv; d.validity = (const uint8_t*)dn;
        r.cols.push_back(d); r.bytes += vb + nb;
    }
    if (rc == BKGPU_OK && cudaStreamSynchronize(st) != cudaSuccess) rc = thread_fail(BKGPU_ENODEV, "bkgpu_region_register: copy failed");
    cudaStreamDestroy(st);
    if (rc != BKGPU_OK) { free_region(r); return rc; }
    std::lock_guard<std::mutex> g(g_region_mu);
    auto key = std::make_pair(device, region_id);
    auto it = g_regions.find(key);
    if (it != g_regions.end()) { free_region(it->second); g_regions.erase(it); }
    g_regions.emplace(key, std::move(r));
    return BKGPU_OK;
}
extern "C" int bkgpu_region_evict(int device, int64_t region_id) {
    std::lock_guard<std::mutex> g(g_region_mu);
    auto it = g_regions.find(std::make_pair(device, region_id));
    if (it == g_regions.end()) return thread_fail(BKGPU_EINVAL, "region %lld is not resident on device %d", (long long)region_id, device);
    cudaSetDevice(device);
    free_region(it->second);
    g_regions.erase(it);
    return BKGPU_OK;
}
extern "C" int bkgpu_region_info(int device, int64_t region_id, int64_t* nrows, size_t* bytes) {
    std::lock_guard<std::mutex> g(g_region_mu);
    auto it = g_regions.find(std::make_pair(device, region_id));
    if (it == g_regions.end()) return thread_fail(BKGPU_EINVAL, "region %lld is not resident on device %d", (long long)region_id, device);
    if (nrows) *nrows = it->second.nrows;
    if (bytes) *bytes = it->second.bytes;
    return BKGPU_OK;
}
// child->get_next() over a resident region: the same as bkgpu_push of its columns with on_device = 1
extern "C" int bkgpu_push_region(bkgpu_plan* p, int64_t region_id) {
    if (!p) return thread_fail(BKGPU_EINVAL, "bkgpu_push_region: NULL plan");
    std::vector<bkgpu_column> cols; int64_t nrows = 0;
    {
        std::lock_guard<std::mutex> g(g_region_mu);
        auto it = g_regions.find(std::make_pair(p->device, region_id));
        if (it == g_regions.end()) return p->fail(BKGPU_EINVAL, "region %lld is not resident on device %d", (long long)region_id, p->device);
        cols = it->second.cols; nrows = it->second.nrows;
    }
    return bkgpu_push(p, cols.data(), (int)cols.size(), nrows, 1);
}

// ------------------------------------------------------------------ partial state
extern "C" int bkgpu_partial_capacity(bkgpu_plan* p, size_t* bytes) {
    if (!p || !bytes) return thread_fail(BKGPU_EINVAL, "bkgpu_partial_capacity: NULL argument");
    if (p->c.n_rb) return p->fail(BKGPU_EUNSUPPORTED, "rb_build_agg has no partial state: bitmaps do not fit the fixed-width partial rows");
    if (p->c.kind == PK_AGG || p->c.kind == PK_JOIN_AGG || p->c.kind == PK_STAR_AGG) {   // (a sketch's registers ride along: HLL_ROW_WORDS per hll_add_agg)
        *bytes = 8 * (1 + (size_t)(p->c.ap.n_keyw + p->c.ap.n_lanes + p->c.ap.n_hll * HLL_ROW_WORDS) * (size_t)eff_pcap(p));
        return BKGPU_OK;
    }
    if (p->c.kind == PK_SORT && p->sort) { *bytes = sort_partial_bytes(p->sort); return BKGPU_OK; }
    return p->fail(BKGPU_EUNSUPPORTED, "plan kind %d has no partial state", p->c.kind);
}
extern "C" int bkgpu_partial_export(bkgpu_plan* p, void* dev_dst, size_t bytes) {
    if (!p || !dev_dst) return thread_fail(BKGPU_EINVAL, "bkgpu_partial_export: NULL argument");
    if (p->state != S_OPEN && p->state != S_FINISHED) return p->fail(BKGPU_ESTATE, "bkgpu_partial_export needs an open plan");
    size_t need = 0; int rc = bkgpu_partial_capacity(p, &need);
    if (rc) return rc;
    if (bytes < need) return p->fail(BKGPU_EINVAL, "partial buffer too small: %zu < %zu", bytes, need);
    CK(p, cudaSetDevice(p->device));
    if (p->c.kind == PK_SORT) return sort_partial_export(p->sort, dev_dst);
    // compact rows (the layout the in-library all-gather ships): [u64 groups][groups x (key words + lane words)]
    CK(p, launch_partial_export_rows(p->gt, p->c.ap, (uint64_t*)dev_dst, eff_pcap(p), p->stream));
    p->stats.kernel_launches += 1;
    uint64_t held = 0; uint32_t ov = 0, hll_ctr[3] = {0, 0, 0};
    CK(p, cudaMemcpyAsync(&held, dev_dst, 8, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaMemcpyAsync(&ov, p->gt.overflow, 4, cudaMemcpyDeviceToHost, p->stream));
    if (p->gt.hll_ctr) CK(p, cudaMemcpyAsync(hll_ctr, p->gt.hll_ctr, 12, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    if (hll_ctr[2]) return p->fail(BKGPU_EINVAL, "MERGE_AGG of hll_add_agg: an input value is not a RAW HLL sketch (\"HYLL\", encoding 255, 16400 bytes)");
    if (hll_ctr[1]) return p->fail(BKGPU_ETOOBIG, "hll_add_agg: more than %u sketches: raise hll_group_capacity", p->gt.hll_cap);
    if (ov) return p->fail(BKGPU_ETOOBIG, "group table overflow (capacity 2^%d slots): raise group_capacity_log2", (int)p->gt.cap_log2);
    if (held > eff_pcap(p)) return p->fail(BKGPU_ETOOBIG, "this rank holds %llu groups, more than partial_capacity=%lld", (unsigned long long)held, (long long)p->partial_cap);
    return BKGPU_OK;
}
extern "C" int bkgpu_partial_merge(bkgpu_plan* p, const void* dev_src, size_t bytes_per_rank, int nranks) {
    if (!p || !dev_src || nranks < 1) return thread_fail(BKGPU_EINVAL, "bkgpu_partial_merge: bad argument");
    if (p->state != S_OPEN && p->state != S_FINISHED) return p->fail(BKGPU_ESTATE, "bkgpu_partial_merge needs an open plan");
    size_t need = 0; int rc = bkgpu_partial_capacity(p, &need);
    if (rc) return rc;
    if (bytes_per_rank != need) return p->fail(BKGPU_EINVAL, "bytes_per_rank %zu != partial capacity %zu", bytes_per_rank, need);
    CK(p, cudaSetDevice(p->device));
    if (p->c.kind == PK_SORT) {
        std::vector<SortOutCol> cols; int64_t rows = 0;
        if ((rc = sort_partial_merge(p->sort, dev_src, nranks, cols, &rows))) return rc;
        set_result(p, cols, rows, nullptr);
        p->stats.rows_returned = rows; p->state = S_FINISHED;
        return BKGPU_OK;
    }
    CK(p, launch_table_init(p->gt, p->c.ap, p->stream, 1));
    CK(p, launch_partial_merge_rows(p->gt, p->c.ap, (const uint64_t*)dev_src, need / 8, eff_pcap(p), nranks, -1 /* fold every segment */, p->d_cursor + 1, p->stream));
    p->fused_last = false;   // (the merged table is read back by k_extract)
    p->stats.kernel_launches += 2;
    void* comm = p->nccl_comm; int nr = p->nranks; p->nccl_comm = nullptr; p->nranks = 1;  // already merged: finalize locally
    rc = agg_finish(p);
    p->nccl_comm = comm; p->nranks = nr;
    if (rc) return rc;
    p->stats.rows_returned = p->result_rows; p->state = S_FINISHED;
    return BKGPU_OK;
}

// ------------------------------------------------------------------ NCCL plumbing
extern "C" int bkgpu_nccl_unique_id(uint8_t id_out[128]) {
    if (!id_out) return thread_fail(BKGPU_EINVAL, "bkgpu_nccl_unique_id: NULL");
    if (nccl_unique_id(id_out) != 0) return thread_fail(BKGPU_ENCCL, "%s", nccl_last_error());
    return BKGPU_OK;
}
extern "C" int bkgpu_nccl_comm_create(void** comm_out, const uint8_t id[128], int nranks, int rank, int device) {
    if (!comm_out || !id) return thread_fail(BKGPU_EINVAL, "bkgpu_nccl_comm_create: NULL");
    if (cudaSetDevice(device) != cudaSuccess) return thread_fail(BKGPU_ENODEV, "cudaSetDevice failed");
    if (nccl_comm_create(comm_out, id, nranks, rank) != 0) return thread_fail(BKGPU_ENCCL, "%s", nccl_last_error());
    return BKGPU_OK;
}
extern "C" void bkgpu_nccl_comm_destroy(void* comm) { if (comm) nccl_comm_destroy(comm); }

// ------------------------------------------------------------------ memory helpers
extern "C" void* bkgpu_host_alloc(size_t bytes) { void* p = nullptr; return cudaHostAlloc(&p, bytes ? bytes : 8, cudaHostAllocDefault) == cudaSuccess ? p : nullptr; }
extern "C" void bkgpu_host_free(void* p) { if (p) cudaFreeHost(p); }
extern "C" void* bkgpu_device_alloc(int device, size_t bytes) {
    void* p = nullptr;
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    return cudaMalloc(&p, bytes ? bytes : 8) == cudaSuccess ? p : nullptr;
}
extern "C" void bkgpu_device_free(int device, void* p) { if (p && cudaSetDevice(device) == cudaSuccess) cudaFree(p); }
extern "C" int bkgpu_memcpy_h2d(int device, void* dst, const void* src, size_t bytes) {
    if (cudaSetDevice(device) != cudaSuccess || cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) return thread_fail(BKGPU_ENODEV, "cudaMemcpy H2D failed");
    return BKGPU_OK;
}
extern "C" int bkgpu_memcpy_d2h(int device, void* dst, const void* src, size_t bytes) {
    if (cudaSetDevice(device) != cudaSuccess || cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return thread_fail(BKGPU_ENODEV, "cudaMemcpy D2H failed");
    return BKGPU_OK;
}

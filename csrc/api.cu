// api.cu — the C ABI of include/bkgpu.h: plan lifecycle (ExecNode::init/open/get_next/close
// inverted into init/open/push/finish/get_next/close), the device buffer cache, batch staging, resident regions and the partial-state entry
// points.  Each plan kind's work is its stage's: the aggregate agg.cu, the hash join join.cu, ORDER BY / filter sort.cu, the window stage
// window.cu; the plan object (bkgpu_plan) is api_state.h.
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
#include "hostcopy.h"

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
    if (rc != BKGPU_OK) { if (text && text_len) snprintf(text, text_len, "%s", err.c_str()); return thread_fail(rc, "%s", err.c_str()); }
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
// the mapped host buffers of the fused extraction (AggState::h_fused) are kept the same way: pinning and unpinning one costs a
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
uint8_t* mapped_take(size_t bytes) { return mapped_cache().take(bytes); }
bool mapped_put(size_t bytes, uint8_t* buf) { return mapped_cache().put(bytes, buf); }

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
    else if (k == "group_capacity_log2") { if (v < 4 || v > 30) return p->fail(BKGPU_EINVAL, "group_capacity_log2 out of range"); p->agg.group_cap_log2 = (int)v; }
    else if (k == "smem_capacity_log2") { if (v < -1 || v > 13) return p->fail(BKGPU_EINVAL, "smem_capacity_log2 out of range"); p->agg.env.smem_cap_log2 = (int)v; }
    else if (k == "batch_capacity") { if (v < 1) return p->fail(BKGPU_EINVAL, "batch_capacity must be positive"); p->batch_capacity = v; }
    else if (k == "chunk_rows") { if (v < 1024) return p->fail(BKGPU_EINVAL, "chunk_rows too small"); p->chunk_rows = (v + 7) & ~7ll; }
    else if (k == "rb_pair_capacity") { if (v < 1024 || v > RADIX_MAX_KEYS) return p->fail(BKGPU_EINVAL, "rb_pair_capacity out of range (1024 .. 2^30 - 1)"); p->agg.rb_cap = v; }
    else if (k == "hll_group_capacity") { if (v < 1 || v > (1 << 20)) return p->fail(BKGPU_EINVAL, "hll_group_capacity out of range (1 .. 2^20)"); p->agg.hll_cap = v; }
    else if (k == "partial_capacity") { if (v < 1) return p->fail(BKGPU_EINVAL, "partial_capacity must be positive"); p->agg.partial_cap = v; }
    else if (k == "force_generic") p->agg.env.force_generic = v != 0;
    else if (k == "lean_fx") p->agg.env.lean_fx = v != 0;
    else if (k == "blocking_sync") p->agg.blocking_sync = (int)v;
    else if (k == "star_expand_capacity") { if (v < 0 || v > 0x7FFFFFFF) return p->fail(BKGPU_EINVAL, "star_expand_capacity out of range"); p->join.star_expand_cap = (int)v; }
    else if (k == "no_lean") p->agg.env.no_lean = v != 0;
    else if (k == "no_fused_probe") p->join.no_fused_probe = v != 0;
    else if (k == "repartition") p->agg.repartition = v != 0;
    else if (k == "no_lean_nulls") p->agg.env.no_lean_nulls = v != 0;
    else if (k == "no_lean_mm") p->agg.env.no_lean_mm = v != 0;
    else if (k == "scalar_tma") p->agg.env.scalar_tma = v != 0;
    else if (k == "region_base") p->region_base = v;
    else return p->fail(BKGPU_EINVAL, "unknown option '%s'", key);
    return BKGPU_OK;
}

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
    for (int i = 0; i < 2; i++) {
        CK(p, cudaEventCreateWithFlags(&p->stage_free[i], cudaEventDisableTiming));
        CK(p, cudaEventCreateWithFlags(&p->stage_ready[i], cudaEventDisableTiming));
    }
    // (refusals that need only the plan and its options: before anything is allocated)
    if (p->c.ap.n_hll && p->agg.repartition)
        return p->fail(BKGPU_EUNSUPPORTED, "hll_add_agg with the repartition merge is outside the GPU path: its sketches travel only with the all-gather of group rows");
    if (p->c.n_rb && p->nccl_comm)
        return p->fail(BKGPU_EUNSUPPORTED, "rb_build_agg with a communicator is outside the GPU path: bitmaps do not travel with the fixed-width partial rows");
    if (p->c.post && p->c.post->kind == PK_WINDOW && p->c.kind != PK_WINDOW && p->agg.repartition)
        return p->fail(BKGPU_EUNSUPPORTED, "a window above an aggregate with the repartition merge is outside the GPU path: each rank would hold only its own groups, "
                       "and a window needs all of them");
    if (p->c.sub && p->nccl_comm)
        return p->fail(BKGPU_EUNSUPPORTED, "a scalar subquery with a communicator is outside the GPU path: the subquery's group table would have to be merged "
                       "across ranks before the first outer row is looked up");
    int rc = upload_in_sets(p);
    if (rc) return rc;
    if (p->c.kind == PK_AGG || p->c.kind == PK_JOIN_AGG || p->c.kind == PK_STAR_AGG) rc = agg_open(p, p->agg, p->c);
    if (!rc && p->c.sub) rc = apply_open(p);
    if (!rc && (p->c.kind == PK_SORT || p->c.kind == PK_FILTER || p->c.kind == PK_WINDOW))   // (a window retains its rows like a full sort)
        rc = sort_open(p, p->c, p->region_base, &p->sort);
    if (!rc && p->c.post) rc = sort_open(p, *p->c.post, 0, &p->post);
    if (!rc && p->c.post && p->c.post->post) rc = sort_open(p, *p->c.post->post, 0, &p->outer);   // (windows above an aggregate: the query's ORDER BY)
    if (rc) return rc;
    p->state = S_OPEN;
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
// at a fraction of the link rate.  The pool (CopyPool, hostcopy.h) is process-wide; plans pushing from several threads take turns on it ----
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
namespace {
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
    bool issued = false;   // a host-to-device copy of the caller's buffers is queued on copy_stream
    rc = [&]() -> int {
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
            issued = true;
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
        return BKGPU_OK;
    }();
    // the caller's host buffers are borrowed for the duration of the call only (bkgpu.h): the last host-to-device copy must have
    // read them before bkgpu_push returns (the kernels read the staging buffers, they may still be running).  That holds on the
    // early returns too — a cancel, a failing stage, a failing CUDA call — since a pinned batch is read in place by the DMA engine.
    if (rc) { if (issued) cudaStreamSynchronize(p->copy_stream); return rc; }
    if (last_ready) CK(p, cudaEventSynchronize(last_ready));
    return BKGPU_OK;
}

static int sort_batch(bkgpu_plan* p, const DevCol* cols, int64_t nrows, int64_t, bool) { return sort_push(p->sort, cols, nrows, &p->stats); }

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
        case PK_AGG: return agg_push(p, cols, ncols, nrows, on_device);
        case PK_JOIN_AGG: case PK_JOIN: case PK_STAR_AGG: return join_push(p, cols, ncols, nrows, on_device);
        case PK_SORT: case PK_FILTER: case PK_WINDOW: return feed(p, p->c.cols, cols, ncols, nrows, on_device, sort_batch);
        default: return p->fail(BKGPU_EUNSUPPORTED, "plan kind %d has no push path yet", p->c.kind);
    }
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
        case PK_AGG: case PK_JOIN_AGG: case PK_STAR_AGG:
            if (p->c.kind == PK_JOIN_AGG && (rc = join_tail(p))) break;
            rc = agg_finish(p);
            if (!rc && p->c.sub) rc = apply_finish(p);
            break;
        case PK_JOIN:   // the outer join's preserved rows, then the sink fragment's result
            if ((rc = join_tail(p)) || (rc = sort_finish(p->post, nullptr, 1, &p->stats, p->c.out_cols.data()))) break;
            p->stats.rows_filtered = 0;
            break;
        case PK_SORT: case PK_FILTER: rc = sort_finish(p->sort, p->nccl_comm, p->nranks, &p->stats, nullptr); break;
        case PK_WINDOW:   // the retained rows through the window stages (window.cu), then the query's ORDER BY when there is one
            if (p->nccl_comm && p->nranks > 1) { rc = p->fail(BKGPU_EUNSUPPORTED, "a window fragment runs on one GPU: multi-GPU merge is implemented for ORDER BY ... LIMIT (top-k) and aggregates"); break; }
            rc = window_finish(p, p->c, p->sort, p->post, &p->stats);
            break;
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
    // cancelled: eos, like the reference's operators — also when the cancel cut the request short before its bkgpu_finish
    if (p->cancelled.load() && (p->state == S_OPEN || p->state == S_FINISHED)) { *eos = 1; *nrows = 0; *ncols = 0; return BKGPU_OK; }
    if (p->state != S_FINISHED) return p->fail(BKGPU_ESTATE, "bkgpu_get_next before bkgpu_finish");
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
        int rc = agg_reset(p, p->agg, p->c);
        if (!rc && p->c.sub) rc = apply_reset(p);
        if (rc) return rc;
    }
    join_reset(p);
    if (p->sort) sort_reset(p->sort);
    if (p->c.kind == PK_JOIN && p->post) sort_reset(p->post);
    if (p->c.kind != PK_WINDOW && p->c.post && p->c.post->kind == PK_WINDOW) {   // windows above an aggregate: their input rows, the query's ORDER BY
        sort_reset(p->post);
        if (p->outer) sort_reset(p->outer);
    }
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
    if (p->post) sort_close(p->post);
    if (p->outer) sort_close(p->outer);
    for (cudaEvent_t e : p->event_pool) cudaEventDestroy(e);
    for (auto& q : p->dev_allocs) if (!dev_cache().put(p->device, q.second, q.first)) cudaFree(q.first);   // (both streams were drained above)
    for (int i = 0; i < 2; i++) { if (p->stage_free[i]) cudaEventDestroy(p->stage_free[i]); if (p->stage_ready[i]) cudaEventDestroy(p->stage_ready[i]); }
    for (int i = 0; i < 2; i++) { for (uint8_t* q : p->bounce[i]) if (q) cudaFreeHost(q); if (p->bounce_done[i]) cudaEventDestroy(p->bounce_done[i]); }
    agg_close(p->agg);
    apply_close(p);
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
    if (p->c.kind == PK_AGG || p->c.kind == PK_JOIN_AGG || p->c.kind == PK_STAR_AGG) { *bytes = agg_partial_bytes(p); return BKGPU_OK; }
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
    return agg_partial_export(p, dev_dst);
}
extern "C" int bkgpu_partial_merge(bkgpu_plan* p, const void* dev_src, size_t bytes_per_rank, int nranks) {
    if (!p || !dev_src || nranks < 1) return thread_fail(BKGPU_EINVAL, "bkgpu_partial_merge: bad argument");
    if (p->state != S_OPEN && p->state != S_FINISHED) return p->fail(BKGPU_ESTATE, "bkgpu_partial_merge needs an open plan");
    size_t need = 0; int rc = bkgpu_partial_capacity(p, &need);
    if (rc) return rc;
    if (bytes_per_rank != need) return p->fail(BKGPU_EINVAL, "bytes_per_rank %zu != partial capacity %zu", bytes_per_rank, need);
    CK(p, cudaSetDevice(p->device));
    if ((rc = p->c.kind == PK_SORT ? sort_partial_merge(p->sort, dev_src, nranks) : agg_partial_merge(p, dev_src, nranks))) return rc;
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

// rb.cu — rb_build_agg's bitmaps, built on the device from the pair buffer the aggregate kernel fills (agg.cu, rb_row).
//
// The reference adds each non-NULL value to a CRoaring bitmap per group (agg_fn_call.cpp:642-651) and ships the bitmap as
// runOptimize() + CRoaring's portable serialization (ExprValue::get_string, expr_value.h:751-760; CRoaring v0.2.66).  A bitmap is a
// function of the set of values alone, so the device collects (group slot, aggregate, value) keys in any order and then:
//   1. sorts them (LSD radix sort, 8 bits per pass; digits on which every key agrees are skipped) and drops duplicates;
//   2. segments them into containers (same slot, aggregate and high 16 bits) and runs (consecutive low halves);
//   3. types each container as add() + runOptimize() leave it: ARRAY up to 4096 values, else BITSET; then RUN when its serialized
//      size 2 + 4 * runs is strictly smaller (than 2 + 2 * card, or than 8192);
//   4. sizes every bitmap, scans the sizes into offsets and writes every bitmap's bytes into one buffer.
// The host copies that buffer and a directory (bitmap id, offset) back.
#include <string.h>
#include <algorithm>
#include "api_state.h"
#include "prims.cuh"
#include "rb.h"

namespace bk {

namespace {

// ---- duplicates ----
__global__ void k_uniq_flags(const uint64_t* k, int64_t n, uint32_t* f) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x)
        f[i] = i == n ? 0u : (i == 0 || k[i] != k[i - 1]) ? 1u : 0u;
}
__global__ void k_uniq_write(const uint64_t* k, int64_t n, const uint32_t* pos, uint64_t* out, unsigned long long* ctr) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (i == 0 || k[i] != k[i - 1]) out[pos[i]] = k[i];
    if (blockIdx.x == 0 && threadIdx.x == 0) *ctr = pos[n];
}

// ---- containers, runs and bitmaps of the sorted distinct keys u[0, m) ----
enum : uint8_t { CT_ARRAY = 1, CT_BITSET = 2, CT_RUN = 3 };
constexpr uint32_t SERIAL_COOKIE_NO_RUNCONTAINER = 12346, SERIAL_COOKIE = 12347, NO_OFFSET_THRESHOLD = 4;

__device__ __forceinline__ bool cont_start(const uint64_t* u, int64_t i) { return i == 0 || (u[i] >> 16) != (u[i - 1] >> 16); }
__device__ __forceinline__ bool run_start(const uint64_t* u, int64_t i) { return cont_start(u, i) || u[i] != u[i - 1] + 1; }
__device__ __forceinline__ void put16(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
__device__ __forceinline__ void put32(uint8_t* p, uint32_t v) { put16(p, v); put16(p + 2, v >> 16); }

// S[i] = container start << 32 | run start (S[m] = 0): its exclusive scan numbers every key's container and run
__global__ void k_seg_flags(const uint64_t* u, int64_t m, uint64_t* s) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= m; i += (int64_t)gridDim.x * blockDim.x)
        s[i] = i == m ? 0ull : ((uint64_t)cont_start(u, i) << 32) | (uint64_t)run_start(u, i);
}
// first key of each container (cst) and run (rst), first run of each container (crun); entry [C] / [R] closes the last one
__global__ void k_seg_mark(const uint64_t* u, int64_t m, const uint64_t* e, uint32_t* cst, uint32_t* crun, uint32_t* rst) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= m; i += (int64_t)gridDim.x * blockDim.x) {
        if (i == m) { const uint64_t c = e[m] >> 32, r = (uint32_t)e[m]; cst[c] = (uint32_t)m; crun[c] = (uint32_t)r; rst[r] = (uint32_t)m; continue; }
        const bool cs = cont_start(u, i), rs = run_start(u, i);
        if (cs) { cst[e[i] >> 32] = (uint32_t)i; crun[e[i] >> 32] = (uint32_t)e[i]; }
        if (rs) rst[(uint32_t)e[i]] = (uint32_t)i;
    }
}
// each container's type after add() + runOptimize(), its payload bytes (psz) and whether it starts a bitmap (bf)
__global__ void k_containers(const uint64_t* u, int64_t nc, const uint32_t* cst, const uint32_t* crun, uint8_t* ctype, uint64_t* psz, uint32_t* bf) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c <= nc; c += (int64_t)gridDim.x * blockDim.x) {
        if (c == nc) { psz[c] = 0; bf[c] = 0; continue; }
        const uint32_t card = cst[c + 1] - cst[c], runs = crun[c + 1] - crun[c];
        uint8_t t;
        if (card <= 4096) t = 2 * runs < card ? CT_RUN : CT_ARRAY;   // 2 + 4 runs < 2 + 2 card (a tie stays ARRAY)
        else t = runs <= 2047 ? CT_RUN : CT_BITSET;                   // 2 + 4 runs < 8192
        ctype[c] = t;
        psz[c] = t == CT_ARRAY ? 2ull * card : t == CT_RUN ? 2ull + 4ull * runs : 8192ull;
        bf[c] = c == 0 || (u[cst[c]] >> 32) != (u[cst[c - 1]] >> 32);
    }
}
// bix(c) = bi[c + 1] - 1 (bi: the exclusive scan of bf): each bitmap's first container, whether it holds a RUN container
__global__ void k_bitmap_start(int64_t nc, const uint32_t* bi, const uint8_t* ctype, uint32_t* bst, uint8_t* bhas) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c <= nc; c += (int64_t)gridDim.x * blockDim.x) {
        if (c == nc) { bst[bi[nc]] = (uint32_t)nc; continue; }
        const uint32_t b = bi[c + 1] - 1;
        if (bi[c + 1] != bi[c]) bst[b] = (uint32_t)c;
        if (ctype[c] == CT_RUN) bhas[b] = 1;
    }
}
// header and total bytes of each bitmap (portable format: ra_portable_serialize), its id (slot << 2 | aggregate)
__device__ __forceinline__ uint32_t bitmap_header(uint32_t size, bool has_run) {
    return has_run ? 4 + (size + 7) / 8 + 4 * size + (size >= NO_OFFSET_THRESHOLD ? 4 * size : 0) : 8 + 8 * size;
}
__global__ void k_bitmap_size(const uint64_t* u, int64_t nc, const uint32_t* bi, const uint32_t* bst, const uint8_t* bhas, const uint64_t* p,
                              const uint32_t* cst, uint32_t* bhdr, uint64_t* bo, uint32_t* bid) {
    const uint32_t nb = bi[nc];
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b <= nc; b += (int64_t)gridDim.x * blockDim.x) {
        if (b >= nb) { bo[b] = 0; continue; }
        const uint32_t hdr = bitmap_header(bst[b + 1] - bst[b], bhas[b] != 0);
        bhdr[b] = hdr;
        bo[b] = hdr + p[bst[b + 1]] - p[bst[b]];
        bid[b] = (uint32_t)(u[cst[bst[b]]] >> 32);
    }
}
// per container: the bitmap's cookie (first container), its (key, card - 1) pair, its offset entry, the run bitmap byte (every eighth
// container), a RUN container's run count; coff = where its payload goes
__global__ void k_headers(const uint64_t* u, int64_t nc, const uint32_t* bi, const uint32_t* bst, const uint8_t* bhas, const uint32_t* bhdr,
                          const uint64_t* bo, const uint64_t* p, const uint32_t* cst, const uint32_t* crun, const uint8_t* ctype, uint8_t* out, uint64_t* coff) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t b = bi[c + 1] - 1, j = (uint32_t)c - bst[b], size = bst[b + 1] - bst[b];
        const bool hr = bhas[b] != 0;
        uint8_t* base = out + bo[b];
        if (j == 0) {
            if (hr) put32(base, SERIAL_COOKIE | ((size - 1) << 16));
            else { put32(base, SERIAL_COOKIE_NO_RUNCONTAINER); put32(base + 4, size); }
        }
        const uint32_t koff = hr ? 4 + (size + 7) / 8 : 8;
        put16(base + koff + 4 * j, (uint32_t)(u[cst[c]] >> 16) & 0xFFFFu);
        put16(base + koff + 4 * j + 2, cst[c + 1] - cst[c] - 1);
        const uint32_t rel = bhdr[b] + (uint32_t)(p[c] - p[bst[b]]);
        if (!hr || size >= NO_OFFSET_THRESHOLD) put32(base + koff + 4 * size + 4 * j, rel);
        if (hr && j % 8 == 0) {
            uint32_t bits = 0;
            for (uint32_t t = 0; t < 8 && j + t < size; t++) if (ctype[c + t] == CT_RUN) bits |= 1u << t;
            base[4 + j / 8] = (uint8_t)bits;
        }
        coff[c] = bo[b] + rel;
        if (ctype[c] == CT_RUN) put16(out + coff[c], crun[c + 1] - crun[c]);
    }
}
// ARRAY: the low halves; RUN: (start, length - 1) per run
__global__ void k_payloads(const uint64_t* u, int64_t m, const uint64_t* e, const uint8_t* ctype, const uint64_t* coff, const uint32_t* cst,
                           const uint32_t* crun, const uint32_t* rst, uint8_t* out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t c = (e[i] >> 32) + (cont_start(u, i) ? 0 : (uint64_t)-1) ;
        const uint32_t low = (uint32_t)u[i] & 0xFFFFu;
        if (ctype[c] == CT_ARRAY) put16(out + coff[c] + 2 * (i - cst[c]), low);
        else if (ctype[c] == CT_RUN && run_start(u, i)) {
            const uint32_t r = (uint32_t)e[i];
            put16(out + coff[c] + 2 + 4 * (r - crun[c]), low);
            put16(out + coff[c] + 4 + 4 * (r - crun[c]), rst[r + 1] - rst[r] - 1);
        }
    }
}
// BITSET: one CTA per container sets its bits in shared memory (bit v % 64 of 64-bit word v / 64, little-endian) and writes the 8192 bytes
__global__ void __launch_bounds__(256) k_bitsets(const uint64_t* u, int64_t nc, const uint32_t* cst, const uint8_t* ctype, const uint64_t* coff, uint8_t* out) {
    __shared__ uint32_t w[2048];
    for (int64_t c = blockIdx.x; c < nc; c += gridDim.x) {
        if (ctype[c] != CT_BITSET) continue;
        for (int t = threadIdx.x; t < 2048; t += blockDim.x) w[t] = 0;
        __syncthreads();
        for (uint32_t i = cst[c] + threadIdx.x; i < cst[c + 1]; i += blockDim.x) { const uint32_t v = (uint32_t)u[i] & 0xFFFFu; atomicOr(&w[v >> 5], 1u << (v & 31)); }
        __syncthreads();
        const uint8_t* src = (const uint8_t*)w;
        for (int t = threadIdx.x; t < 8192; t += blockDim.x) out[coff[c] + t] = src[t];
        __syncthreads();
    }
}

}  // namespace

// scratch buffer `slot` of the plan's rb state, at least `bytes` long
static int rb_buf(bkgpu_plan* p, int slot, size_t bytes, void** out) {
    int rc = ensure_buf(p, &p->agg.rb.scratch[slot], &p->agg.rb.scratch_cap[slot], std::max<size_t>(bytes, 8));
    *out = p->agg.rb.scratch[slot];
    return rc;
}
template <typename T> static T d2h(bkgpu_plan* p, const T* src, int* rc) {
    T v{};
    cudaError_t e = cudaMemcpyAsync(&v, src, sizeof(T), cudaMemcpyDeviceToHost, p->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(p->stream);
    if (e != cudaSuccess) *rc = p->cuda_fail(e, "rb_build_agg: device-to-host copy");
    return v;
}

// sort keys [0, n) of the pair buffer: p->agg.rb.keys then points at the sorted keys (the sort's second buffer is p->agg.rb.alt)
static int rb_sort(bkgpu_plan* p, int64_t n) {
    uint64_t* keys[2] = {p->agg.rb.keys, p->agg.rb.alt};
    const int r = radix_sort(p, keys, nullptr, 0, n, p->agg.rb.sort, &p->stats, nullptr);
    if (r < 0) return r;
    if (r) std::swap(p->agg.rb.keys, p->agg.rb.alt);
    return BKGPU_OK;
}

int rb_compact(bkgpu_plan* p, uint64_t* n_out) {
    int rc = BKGPU_OK;
    const uint64_t n = d2h(p, p->agg.rb.ctr, &rc);
    if (rc) return rc;
    if (n > p->agg.rb.cap)
        return p->fail(BKGPU_ETOOBIG, "rb_build_agg: more than %llu (group, value) pairs in one batch: raise rb_pair_capacity", (unsigned long long)p->agg.rb.cap);
    if ((rc = rb_sort(p, (int64_t)n))) return rc;
    uint32_t *flags, *sums;
    // (the flags reuse the sort's look-back status buffer: the sort is done with it)
    if ((rc = ensure_buf(p, &p->agg.rb.sort.status, &p->agg.rb.sort.status_cap, (n + 1) * 4))) return rc;
    flags = (uint32_t*)p->agg.rb.sort.status;
    if ((rc = rb_buf(p, 0, (size_t)scan_scratch((int64_t)n + 1) * 4, (void**)&sums))) return rc;
    const int g = grid_for((int64_t)n + 1, p->sm_count, 16);
    k_uniq_flags<<<g, 256, 0, p->stream>>>(p->agg.rb.keys, (int64_t)n, flags);
    CK(p, cudaGetLastError());
    CK(p, scan_excl(flags, (int64_t)n + 1, sums, p->sm_count, p->stream));
    k_uniq_write<<<g, 256, 0, p->stream>>>(p->agg.rb.keys, (int64_t)n, flags, p->agg.rb.alt, p->agg.rb.ctr);
    CK(p, cudaGetLastError());
    std::swap(p->agg.rb.keys, p->agg.rb.alt);
    p->stats.kernel_launches += 4;
    *n_out = d2h(p, p->agg.rb.ctr, &rc);
    return rc;
}

int rb_build(bkgpu_plan* p) {
    uint64_t m64 = 0;
    int rc = rb_compact(p, &m64);
    if (rc) return rc;
    const int64_t m = (int64_t)m64;
    const cudaStream_t s = p->stream;
    const int sm = p->sm_count;
    p->agg.rb.bid.clear(); p->agg.rb.off.assign(1, 0);
    if (m == 0) return BKGPU_OK;
    const uint64_t* u = p->agg.rb.keys;
    uint64_t* e = p->agg.rb.alt;   // (cap + 1 words: room for the scan's closing entry)
    uint64_t* sums64;
    if ((rc = rb_buf(p, 0, (size_t)scan_scratch(m + 1) * 8, (void**)&sums64))) return rc;
    k_seg_flags<<<grid_for(m + 1, sm, 16), 256, 0, s>>>(u, m, e);
    CK(p, cudaGetLastError());
    CK(p, scan_excl(e, m + 1, sums64, sm, s));
    const uint64_t tot = d2h(p, e + m, &rc);
    if (rc) return rc;
    const int64_t nc = (int64_t)(tot >> 32), nr = (int64_t)(uint32_t)tot;
    uint32_t *cst, *crun, *rst, *bi, *bst, *bhdr, *bid;
    uint8_t *ctype, *bhas, *out;
    uint64_t *psz, *coff, *bo;
    if ((rc = rb_buf(p, 1, (size_t)(nc + 1) * 4, (void**)&cst)) || (rc = rb_buf(p, 2, (size_t)(nc + 1) * 4, (void**)&crun)) ||
        (rc = rb_buf(p, 3, (size_t)(nr + 1) * 4, (void**)&rst)) || (rc = rb_buf(p, 4, (size_t)nc, (void**)&ctype)) ||
        (rc = rb_buf(p, 5, (size_t)(nc + 1) * 8, (void**)&psz)) || (rc = rb_buf(p, 6, (size_t)(nc + 1) * 4, (void**)&bi)) ||
        (rc = rb_buf(p, 7, (size_t)nc * 8, (void**)&coff)) || (rc = rb_buf(p, 8, (size_t)(nc + 1) * 4, (void**)&bst)) ||
        (rc = rb_buf(p, 9, (size_t)(nc + 1), (void**)&bhas)) || (rc = rb_buf(p, 10, (size_t)(nc + 1) * 4, (void**)&bhdr)) ||
        (rc = rb_buf(p, 11, (size_t)(nc + 1) * 8, (void**)&bo)) || (rc = rb_buf(p, 12, (size_t)(nc + 1) * 4, (void**)&bid)) ||
        (rc = rb_buf(p, 0, (size_t)scan_scratch(std::max(m, nc) + 1) * 8, (void**)&sums64)))
        return rc;
    k_seg_mark<<<grid_for(m + 1, sm, 16), 256, 0, s>>>(u, m, e, cst, crun, rst);
    k_containers<<<grid_for(nc + 1, sm, 16), 256, 0, s>>>(u, nc, cst, crun, ctype, psz, bi);
    CK(p, cudaGetLastError());
    CK(p, scan_excl(psz, nc + 1, sums64, sm, s));
    CK(p, scan_excl(bi, nc + 1, (uint32_t*)sums64, sm, s));
    CK(p, cudaMemsetAsync(bhas, 0, (size_t)(nc + 1), s));
    k_bitmap_start<<<grid_for(nc + 1, sm, 16), 256, 0, s>>>(nc, bi, ctype, bst, bhas);
    k_bitmap_size<<<grid_for(nc + 1, sm, 16), 256, 0, s>>>(u, nc, bi, bst, bhas, psz, cst, bhdr, bo, bid);
    CK(p, cudaGetLastError());
    CK(p, scan_excl(bo, nc + 1, sums64, sm, s));
    uint32_t nb = 0; uint64_t total = 0;
    CK(p, cudaMemcpyAsync(&nb, bi + nc, 4, cudaMemcpyDeviceToHost, s));
    CK(p, cudaMemcpyAsync(&total, bo + nc, 8, cudaMemcpyDeviceToHost, s));
    CK(p, cudaStreamSynchronize(s));
    if ((rc = rb_buf(p, 13, (size_t)total, (void**)&out))) return rc;
    k_headers<<<grid_for(nc, sm, 16), 256, 0, s>>>(u, nc, bi, bst, bhas, bhdr, bo, psz, cst, crun, ctype, out, coff);
    k_payloads<<<grid_for(m, sm, 16), 256, 0, s>>>(u, m, e, ctype, coff, cst, crun, rst, out);
    k_bitsets<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>(nc, (int64_t)sm * 8)), 256, 0, s>>>(u, nc, cst, ctype, coff, out);
    CK(p, cudaGetLastError());
    p->stats.kernel_launches += 16;
    // the finished bytes and the directory back to the host: bitmap ids ascend (the keys were sorted), offsets close with the total
    p->agg.rb.bid.resize(nb); p->agg.rb.off.resize((size_t)nb + 1);
    if (p->agg.rb.bytes_cap < total) {
        if (p->agg.rb.bytes) cudaFreeHost(p->agg.rb.bytes);
        p->agg.rb.bytes = nullptr; p->agg.rb.bytes_cap = 0;
        CK(p, cudaHostAlloc((void**)&p->agg.rb.bytes, total + total / 4, cudaHostAllocDefault));
        p->agg.rb.bytes_cap = total + total / 4;
    }
    CK(p, cudaMemcpyAsync(p->agg.rb.bid.data(), bid, (size_t)nb * 4, cudaMemcpyDeviceToHost, s));
    CK(p, cudaMemcpyAsync(p->agg.rb.off.data(), bo, ((size_t)nb + 1) * 8, cudaMemcpyDeviceToHost, s));
    CK(p, cudaMemcpyAsync(p->agg.rb.bytes, out, total, cudaMemcpyDeviceToHost, s));
    CK(p, cudaStreamSynchronize(s));
    p->stats.d2h_bytes += (int64_t)(total + (size_t)nb * 12 + 8);
    return BKGPU_OK;
}

}  // namespace bk

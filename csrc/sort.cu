// sort.cu — K5 (ORDER BY / top-k) and K1 (filter-only stream compaction) for sm_90a.
//
// Replaces SortNode::open + Sorter / TopNSorter (src/exec/sort_node.cpp:278-346, src/runtime/sorter.cpp:54-114,
// src/runtime/topn_sorter.cpp:25-103) and the row-copy half of FilterNode::get_next (src/exec/filter_node.cpp:736-795).
//
// Ordering is the reference's MemRowCompare (src/mem_row/mem_row_compare.cpp:18-38) made total: every row
// carries the composite (class, key image, arrival index) where class orders NULL keys first / last
// (is_null_first), the key image is an order-preserving 64-bit transform (descending = complemented)
// and the arrival index breaks ties the way TopNSorter does (include/runtime/topn_sorter.h:96-106).
//
// ORDER BY ... LIMIT k (one key): selection, not sorting.  Per batch:
//   sample 4096 random positions -> threshold at a rank that leaves >= k rows below it with overwhelming
//   probability -> ONE pass over the key column compacts the candidates (warp-ballot compaction, 8 B/row) ->
//   the same step recurses on the shrinking candidate arrays until <= 8192 remain -> one CTA sorts them in
//   shared memory together with the k rows kept from earlier batches -> payload columns are gathered for
//   the k survivors only.
// ORDER BY without LIMIT / several keys: LSD radix sort (8 bits per pass, stable) of (key image, row id),
//   least significant ORDER BY key first, then a gather of every column.
// Filter-only fragments: predicate -> ordered compaction (block scan) -> gather, honouring LIMIT in input order.
#include "sort.h"
#include <algorithm>
#include <string.h>
#include "api_state.h"
#include "dev_common.cuh"
#include "interp.cuh"
#include "nccl_dl.h"
#include "prims.cuh"
#include "sort_key.h"   // key_image: the order-preserving 64-bit image (ascending); DESC complements it

namespace bk {

namespace {

constexpr int SMALL_N = 8192;        // one CTA sorts this many composite keys in shared memory
constexpr int SAMPLE_N = 4096;

struct KeySpec {       // how a row's sort key is obtained on the device
    int direct;        // 1: plain column `col` of class `vclass`; 0: program output register `out_reg`
    int col, vclass, out_reg;
    int desc;          // ORDER BY ... DESC
    int pred_out;      // predicate register (-1 = none); generic path only
};

struct RowArgs {
    DevCol cols[MAX_COLS];
    int32_t n_cols;
    int64_t nrows;
    uint64_t row_base;   // arrival index of row 0 of this batch
    Program prog;
    KeySpec key;
};

// cls: 0 = row filtered out, 1 = key present, 2 = key is NULL
__device__ __forceinline__ int row_key(const RowArgs& a, int64_t row, uint64_t& image) {
    if (a.key.direct) {
        const DevCol& c = a.cols[a.key.col];
        if (elem_is_null(c, row)) { image = 0; return 2; }
        image = key_image(load_elem(c, row), a.key.vclass, a.key.desc);
        return 1;
    }
    uint64_t out[8]; uint32_t out_null;
    run_program(a.prog, a.cols, row, out, out_null);
    if (a.key.pred_out >= 0 && (((out_null >> a.key.pred_out) & 1u) || out[a.key.pred_out] == 0)) return 0;
    if ((out_null >> a.key.out_reg) & 1u) { image = 0; return 2; }
    image = key_image(out[a.key.out_reg], a.key.vclass, a.key.desc);
    return 1;
}

__device__ __forceinline__ bool comp_le(uint64_t k, uint64_t i, uint64_t tk, uint64_t ti) { return k < tk || (k == tk && i <= ti); }
__device__ __forceinline__ bool comp_lt(uint64_t k, uint64_t i, uint64_t tk, uint64_t ti) { return k < tk || (k == tk && i < ti); }

__device__ __forceinline__ uint64_t mix64d(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31);
}

// ---- level-1 kernels: straight from the batch columns ----
// sample: position i of SAMPLE_N is drawn uniformly inside its stratum [i*n/S, (i+1)*n/S)
__global__ void k_sample_rows(RowArgs a, int want_cls, uint64_t* skey, uint64_t* sidx, uint32_t* scount, uint64_t salt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= SAMPLE_N) return;
    const int64_t lo = (int64_t)(((__int128)i * a.nrows) / SAMPLE_N), hi = (int64_t)(((__int128)(i + 1) * a.nrows) / SAMPLE_N);
    if (hi <= lo) return;
    const int64_t row = lo + (int64_t)(mix64d(salt + i) % (uint64_t)(hi - lo));
    uint64_t img;
    if (row_key(a, row, img) != want_cls) return;
    const uint32_t pos = atomicAdd(scount, 1u);
    skey[pos] = img; sidx[pos] = a.row_base + (uint64_t)row;
}

// compaction of the rows whose composite key is <= (tk, ti): warp-ballot positions, one atomic per warp
__global__ void __launch_bounds__(256) k_collect_rows(RowArgs a, int want_cls, const uint64_t* thr, uint64_t* okey, uint64_t* oidx,
                                                      uint32_t* ocount, uint32_t cap, uint32_t* class_count) {
    const int lane = threadIdx.x & 31;
    const uint64_t tk = thr[0], ti = thr[1];   // threshold produced on the device by k_sort_small: no host round trip
    uint32_t seen = 0;
    for (int64_t base = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x - lane); base < a.nrows; base += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = base + lane;
        uint64_t img = 0; bool take = false;
        if (row < a.nrows) {
            const int cls = row_key(a, row, img);
            if (cls == want_cls) { seen++; take = comp_le(img, a.row_base + (uint64_t)row, tk, ti); }
        }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, take);
        if (b) {
            uint32_t wbase = 0;
            if (lane == 0) wbase = atomicAdd(ocount, (uint32_t)__popc(b));
            wbase = __shfl_sync(0xFFFFFFFFu, wbase, 0);
            const uint32_t pos = wbase + __popc(b & ((1u << lane) - 1u));
            if (take && pos < cap) { okey[pos] = img; oidx[pos] = a.row_base + (uint64_t)row; }
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) seen += __shfl_xor_sync(0xFFFFFFFFu, seen, d);
    if (lane == 0 && seen && class_count) atomicAdd(class_count, seen);
}

// level 1 for the direct shape (plain NULL-free key column, config C5): four keys per lane and load (two LDG.128 / one LDG.128),
// two loads in flight; candidates are rare (~1 % of the rows), so the compaction slow path is off the hot loop
template <int KEY_BYTES>
__global__ void __launch_bounds__(256) k_collect_rows_vec(RowArgs a, const uint64_t* thr, uint64_t* okey, uint64_t* oidx, uint32_t* ocount,
                                                          uint32_t cap, uint32_t* class_count) {
    // candidates are staged per CTA in shared memory and leave with ONE global atomic per CTA: ~1M candidates
    // hammering a single global counter would dominate the pass
    constexpr uint32_t STAGE = 2048;
    __shared__ uint64_t s_key[STAGE], s_idx[STAGE];
    __shared__ uint32_t s_n, s_base;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const uint64_t tk = thr[0], ti = thr[1];
    const DevCol& c = a.cols[a.key.col];
    const int vclass = a.key.vclass, desc = a.key.desc;
    const bool sext = c.stype == ST_I32;
    const int64_t nquads = a.nrows >> 2;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    auto emit = [&](uint64_t img, uint64_t idx) {
        const uint32_t pos = atomicAdd(&s_n, 1u);
        if (pos < STAGE) { s_key[pos] = img; s_idx[pos] = idx; }
        else { const uint32_t g = atomicAdd(ocount, 1u); if (g < cap) { okey[g] = img; oidx[g] = idx; } }   // stage full: rare
    };
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < nquads; q += 2 * stride) {
        uint64_t v[8];
        const bool second = q + stride < nquads;
        if (KEY_BYTES == 8) {
            const U64x4 r0 = ldg256_u64((const uint8_t*)c.values + q * 32);
#pragma unroll
            for (int j = 0; j < 4; j++) v[j] = r0.v[j];
            if (second) { const U64x4 r1 = ldg256_u64((const uint8_t*)c.values + (q + stride) * 32);
#pragma unroll
                for (int j = 0; j < 4; j++) v[4 + j] = r1.v[j]; }
        } else {
            const U32x4 r0 = ldg128_u32((const uint8_t*)c.values + q * 16);
#pragma unroll
            for (int j = 0; j < 4; j++) v[j] = sext ? (uint64_t)(int64_t)(int32_t)r0.v[j] : (uint64_t)r0.v[j];
            if (second) { const U32x4 r1 = ldg128_u32((const uint8_t*)c.values + (q + stride) * 16);
#pragma unroll
                for (int j = 0; j < 4; j++) v[4 + j] = sext ? (uint64_t)(int64_t)(int32_t)r1.v[j] : (uint64_t)r1.v[j]; }
        }
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (j >= 4 && !second) break;
            const uint64_t img = key_image(v[j], vclass, desc);
            if (img > tk) continue;                                    // the common case: not a candidate
            const uint64_t idx = a.row_base + (uint64_t)((j < 4 ? q : q + stride) * 4 + (j & 3));
            if (comp_le(img, idx, tk, ti)) emit(img, idx);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (a.nrows & 3)) {   // ragged tail
        const int64_t row = (a.nrows & ~(int64_t)3) + threadIdx.x;
        const uint64_t img = key_image(load_elem(c, row), vclass, desc);
        if (comp_le(img, a.row_base + (uint64_t)row, tk, ti)) emit(img, a.row_base + (uint64_t)row);
    }
    __syncthreads();
    const uint32_t n = min(s_n, STAGE);
    if (threadIdx.x == 0) s_base = n ? atomicAdd(ocount, n) : 0;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) { const uint32_t g = s_base + i; if (g < cap) { okey[g] = s_key[i]; oidx[g] = s_idx[i]; } }
    if (blockIdx.x == 0 && threadIdx.x == 0 && class_count) atomicAdd(class_count, (uint32_t)min(a.nrows, (int64_t)0xFFFFFFFFll));  // no NULLs, no filter: every row is of this class
}

// ---- level >= 2 kernels: on (key, idx) candidate arrays ----
__global__ void k_sample_pairs(const uint64_t* key, const uint64_t* idx, const uint32_t* n_ptr, uint32_t cap, uint64_t* skey, uint64_t* sidx, uint32_t* scount, uint64_t salt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= SAMPLE_N) return;
    const uint32_t n = min(*n_ptr, cap);
    const uint64_t lo = (uint64_t)i * n / SAMPLE_N, hi = (uint64_t)(i + 1) * n / SAMPLE_N;
    if (hi <= lo) return;
    const uint64_t p = lo + mix64d(salt + i) % (hi - lo);
    const uint32_t pos = atomicAdd(scount, 1u);
    skey[pos] = key[p]; sidx[pos] = idx[p];
}
__global__ void __launch_bounds__(256) k_collect_pairs(const uint64_t* key, const uint64_t* idx, const uint32_t* n_ptr, const uint64_t* thr,
                                                       uint64_t* okey, uint64_t* oidx, uint32_t* ocount, uint32_t cap) {
    const int lane = threadIdx.x & 31;
    const uint32_t n = min(*n_ptr, cap);
    const uint64_t tk = thr[0], ti = thr[1];
    for (uint32_t base = blockIdx.x * blockDim.x + threadIdx.x - lane; base < n; base += gridDim.x * blockDim.x) {
        const uint32_t i = base + lane;
        const bool take = i < n && comp_le(key[i], idx[i], tk, ti);
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, take);
        if (b) {
            uint32_t wbase = 0;
            if (lane == 0) wbase = atomicAdd(ocount, (uint32_t)__popc(b));
            wbase = __shfl_sync(0xFFFFFFFFu, wbase, 0);
            const uint32_t pos = wbase + __popc(b & ((1u << lane) - 1u));
            if (take && pos < cap) { okey[pos] = key[i]; oidx[pos] = idx[i]; }
        }
    }
}

// one CTA: bitonic sort of n <= SMALL_N composite keys in shared memory (ascending); optionally reads a
// second segment (the rows kept from earlier batches).  Writes the first `keep` entries and the r-th (0-based) one.
__global__ void __launch_bounds__(1024) k_sort_small(const uint64_t* k1, const uint64_t* i1, const uint32_t* n1p, uint32_t n1max,
                                                     const uint64_t* k2, const uint64_t* i2, uint32_t n2,
                                                     uint64_t* okey, uint64_t* oidx, uint32_t keep, uint32_t* out_n,
                                                     uint32_t rank, uint64_t* rank_out,
                                                     const uint32_t* pop_ptr, uint32_t k_want, uint32_t widen, uint32_t room, const uint64_t* cap_thr) {
    extern __shared__ __align__(16) unsigned char sm[];
    uint64_t* sk = (uint64_t*)sm; uint64_t* si = sk + SMALL_N;
    uint32_t n1 = n1p ? *n1p : n1max; if (n1 > n1max) n1 = n1max;
    const uint32_t n = n1 + n2;
    uint32_t m = 1; while (m < n) m <<= 1; if (m < 2) m = 2;
    for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
        if (i < n1) { sk[i] = k1[i]; si[i] = i1[i]; }
        else if (i < n) { sk[i] = k2[i - n1]; si[i] = i2[i - n1]; }
        else { sk[i] = ~0ull; si[i] = ~0ull; }
    }
    __syncthreads();
    for (uint32_t size = 2; size <= m; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < (m >> 1); t += blockDim.x) {
                const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const uint64_t ka = sk[lo], ia = si[lo], kb = sk[hi], ib = si[hi];
                const bool a_gt_b = comp_lt(kb, ib, ka, ia);
                if (a_gt_b == up) { sk[lo] = kb; si[lo] = ib; sk[hi] = ka; si[hi] = ia; }
            }
            __syncthreads();
        }
    }
    const uint32_t nk = n < keep ? n : keep;
    if (okey) for (uint32_t i = threadIdx.x; i < nk; i += blockDim.x) { okey[i] = sk[i]; oidx[i] = si[i]; }
    if (threadIdx.x == 0) {
        if (out_n) *out_n = nk;
        if (rank_out) {
            // threshold for the next compaction: the sample (n entries of a population of *pop_ptr) at a rank that
            // leaves >= k_want population members below it with overwhelming probability; +inf when the population
            // already fits `room` or the sample is too small to say anything
            uint64_t tk = ~0ull, ti = ~0ull;
            uint32_t r = rank;
            if (pop_ptr) {
                const double pop = (double)*pop_ptr;
                if (pop <= (double)room) r = 0xFFFFFFFFu;
                else { double w = ((double)k_want * (double)SAMPLE_N / pop * 1.5 + 32.0) * (double)widen; r = w >= (double)(SAMPLE_N - 1) ? 0xFFFFFFFFu : (uint32_t)w; }
            }
            if (n > 0 && r < n) { tk = sk[r]; ti = si[r]; }
            if (cap_thr && comp_lt(cap_thr[0], cap_thr[1], tk, ti)) { tk = cap_thr[0]; ti = cap_thr[1]; }   // never looser than the k-th row kept so far
            rank_out[0] = tk; rank_out[1] = ti; rank_out[2] = n;
        }
    }
}

// one CTA: the r-th smallest (0-based) of n <= SAMPLE_N composite keys by radix selection — most significant byte
// first over the 16 bytes of (key, idx), a 256-bin shared histogram per byte, stopping as soon as the selected bin
// holds one element (random 64-bit keys: 2 rounds).  Same threshold rules as k_sort_small's rank output; replaces
// a full bitonic sort of the sample on the top-k chain.
__global__ void __launch_bounds__(1024) k_select_rank(const uint64_t* key, const uint64_t* idx, const uint32_t* np, uint32_t nmax,
                                                      uint32_t rank, uint64_t* rank_out,
                                                      const uint32_t* pop_ptr, uint32_t k_want, uint32_t widen, uint32_t room, const uint64_t* cap_thr) {
    __shared__ uint32_t hist[256];
    __shared__ uint32_t s_bin, s_rank, s_cnt;
    __shared__ uint64_t s_res[2];
    constexpr int PER = SAMPLE_N / 1024;
    uint32_t n = *np; if (n > nmax) n = nmax; if (n > (uint32_t)SAMPLE_N) n = SAMPLE_N;
    uint32_t r = rank;
    if (pop_ptr) {
        const double pop = (double)*pop_ptr;
        if (pop <= (double)room) r = 0xFFFFFFFFu;
        else { double w = ((double)k_want * (double)SAMPLE_N / pop * 1.5 + 32.0) * (double)widen; r = w >= (double)(SAMPLE_N - 1) ? 0xFFFFFFFFu : (uint32_t)w; }
    }
    if (threadIdx.x == 0) { s_res[0] = ~0ull; s_res[1] = ~0ull; }
    if (n > 0 && r < n) {   // (uniform across the CTA)
        uint64_t k[PER], ix[PER]; uint32_t alive = 0;
#pragma unroll
        for (int e = 0; e < PER; e++) {
            const uint32_t i = threadIdx.x + e * 1024;
            k[e] = 0; ix[e] = 0;
            if (i < n) { k[e] = key[i]; ix[e] = idx[i]; alive |= 1u << e; }
        }
        uint32_t rr = r;
        for (int byte = 15; byte >= 0; byte--) {
            if (threadIdx.x < 256) hist[threadIdx.x] = 0;
            __syncthreads();
            uint32_t dig[PER];
#pragma unroll
            for (int e = 0; e < PER; e++) {
                dig[e] = (uint32_t)((byte >= 8 ? k[e] >> ((byte - 8) * 8) : ix[e] >> (byte * 8)) & 255ull);
                if ((alive >> e) & 1u) atomicAdd(&hist[dig[e]], 1u);
            }
            __syncthreads();
            if (threadIdx.x < 32) {   // warp 0: the bin that holds rank rr
                uint32_t h[8], sum = 0;
#pragma unroll
                for (int j = 0; j < 8; j++) { h[j] = hist[threadIdx.x * 8 + j]; sum += h[j]; }
                uint32_t incl = sum;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) { const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)threadIdx.x >= d) incl += o; }
                uint32_t cum = incl - sum;
                if (rr >= cum && rr < incl) {
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        if (rr < cum + h[j]) { s_bin = threadIdx.x * 8 + j; s_rank = rr - cum; s_cnt = h[j]; break; }
                        cum += h[j];
                    }
                }
            }
            __syncthreads();
            const uint32_t bin = s_bin;
#pragma unroll
            for (int e = 0; e < PER; e++) if (dig[e] != bin) alive &= ~(1u << e);
            rr = s_rank;
            if (s_cnt == 1 || byte == 0) break;
        }
#pragma unroll
        for (int e = 0; e < PER; e++) if ((alive >> e) & 1u) { s_res[0] = k[e]; s_res[1] = ix[e]; }   // one element (or identical ones)
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t tk = s_res[0], ti = s_res[1];
        uint64_t capped = 0;
        if (cap_thr && comp_lt(cap_thr[0], cap_thr[1], tk, ti)) { tk = cap_thr[0]; ti = cap_thr[1]; capped = 1ull << 62; }   // never looser than the k-th row kept so far
        rank_out[0] = tk; rank_out[1] = ti; rank_out[2] = (uint64_t)n | capped;   // bit 62: the threshold in force is the pool's k-th key
    }
}

// ---- payload: gather rows of the current batch / move rows kept from earlier batches ----
__global__ void k_gather_topk(GatherArgs g, const uint64_t* idx, const uint32_t* np) {
    const uint32_t n = *np;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint64_t id = idx[i];
        const bool from_batch = g.nrows > 0 && id >= g.row_base && id < g.row_base + (uint64_t)g.nrows;
        int64_t src = -1;
        if (from_batch) src = (int64_t)(id - g.row_base);
        else {  // binary search in the previous survivors (sorted by composite key, not by idx): linear scan is fine for k rows
            for (uint32_t j = 0; j < g.old_n; j++) if (g.old_idx[j] == id) { src = j; break; }
        }
        for (int c = 0; c < g.n_cols; c++) {
            const int eb = g.cols[c].stype == ST_U8 ? 1 : (g.cols[c].stype == ST_BLOB16 ? 16 : ((g.cols[c].stype == ST_I32 || g.cols[c].stype == ST_U32 || g.cols[c].stype == ST_F32) ? 4 : 8));
            const uint8_t* sv; uint8_t isnull;
            if (from_batch) { sv = (const uint8_t*)g.cols[c].values + (size_t)src * eb; isnull = elem_is_null(g.cols[c], src) ? 1 : 0; }
            else { sv = g.old_vals[c] + (size_t)src * eb; isnull = g.old_null[c][src]; }
            uint8_t* dv = g.dst_vals[c] + (size_t)i * eb;
            for (int b = 0; b < eb; b++) dv[b] = sv[b];
            g.dst_null[c][i] = isnull;
        }
    }
}

// ---- filter-only: ordered compaction.  Pass 1 counts per block, pass 2 (after a scan of the counts) writes. ----
__global__ void __launch_bounds__(256) k_filter_count(RowArgs a, uint32_t* block_counts, int64_t rows_per_block) {
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block, r1 = min(r0 + rows_per_block, a.nrows);
    uint32_t cnt = 0;
    for (int64_t row = r0 + threadIdx.x; row < r1; row += blockDim.x) {
        uint64_t img; const int cls = a.key.pred_out < 0 ? 1 : row_key(a, row, img);
        cnt += cls != 0;
    }
    __shared__ uint32_t s[8];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, d);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) { uint32_t t = 0; for (int i = 0; i < 8; i++) t += s[i]; block_counts[blockIdx.x] = t; }
}
__global__ void __launch_bounds__(256) k_filter_write(RowArgs a, const uint32_t* block_offsets, int64_t rows_per_block, uint32_t* sel, uint64_t out_base, uint64_t cap) {
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block, r1 = min(r0 + rows_per_block, a.nrows);
    __shared__ uint32_t warp_cnt[8];
    __shared__ uint32_t running;
    if (threadIdx.x == 0) running = block_offsets[blockIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t base = r0; base < r1; base += blockDim.x) {
        const int64_t row = base + threadIdx.x;
        bool take = false;
        if (row < r1) { uint64_t img; take = a.key.pred_out < 0 ? true : row_key(a, row, img) != 0; }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, take);
        if (lane == 0) warp_cnt[warp] = __popc(b);
        __syncthreads();
        uint32_t before = running;
        for (int w = 0; w < warp; w++) before += warp_cnt[w];
        const uint64_t pos = out_base + before + __popc(b & ((1u << lane) - 1u));
        if (take && pos < cap) sel[pos] = (uint32_t)row;
        __syncthreads();
        if (threadIdx.x == 0) { uint32_t t = 0; for (int w = 0; w < 8; w++) t += warp_cnt[w]; running += t; }
        __syncthreads();
    }
}
// ---- full sort: materialise (image, row id), LSD radix sort, gather ----
// mode 0: order-preserving image of the key (NULL -> 0); mode 1: the NULL rank (0 sorts first) — sorted by one
// extra radix pass AFTER the eight value passes so NULL keys come strictly first / last (is_null_first)
__global__ void k_sort_images(RowArgs a, int key_reg, int vclass, int desc, int null_first, int mode, uint64_t* img, uint32_t* rid) {
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < a.nrows; row += (int64_t)gridDim.x * blockDim.x) {
        uint64_t out[8]; uint32_t out_null;
        run_program(a.prog, a.cols, row, out, out_null);
        const bool isnull = (out_null >> key_reg) & 1u;
        if (mode == 0) img[row] = isnull ? 0ull : key_image(out[key_reg], vclass, desc);
        else img[row] = isnull ? (null_first ? 0ull : 1ull) : (null_first ? 1ull : 0ull);
        if (rid) rid[row] = (uint32_t)row;
    }
}
// key image of a plain column key, without the expression interpreter
__global__ void k_sort_images_direct(DevCol c, int64_t n, int vclass, int desc, uint64_t* img) {
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x)
        img[row] = elem_is_null(c, row) ? 0ull : key_image(load_elem(c, row), vclass, desc);
}
__global__ void k_rs_gather_u64(const uint64_t* src, const uint32_t* ids, uint64_t* dst, uint32_t n) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[ids[i]];
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------
struct Pool {               // the k best rows seen so far of one class (keys present / NULL keys)
    uint64_t* key[2] = {nullptr, nullptr}; uint64_t* idx[2] = {nullptr, nullptr};
    uint8_t* vals[2][MAX_COLS] = {}; uint8_t* nulls[2][MAX_COLS] = {};
    int cur = 0; uint32_t n = 0;
};

struct SortState {
    bkgpu_plan* p = nullptr;        // the owning plan: its allocator, stream and SM count
    const Compiled* c = nullptr;    // the fragment, owned by the plan
    int ncols = 0;
    int64_t k = -1;                 // rows to keep; -1 = all
    uint64_t row_base = 0, region_base = 0;
    bool topk = false;              // single key + limit: selection path
    bool used_vec = false;
    Pool pool[2];
    // scratch for selection
    uint64_t *cand_key[2] = {nullptr, nullptr}, *cand_idx[2] = {nullptr, nullptr}; uint32_t cand_cap = 0;
    uint64_t *samp_key = nullptr, *samp_idx = nullptr;
    uint32_t* d_counts = nullptr;   // [0] sample count, [1] candidate count A, [2] candidate count B, [3] class count, [4] pool out n
    uint64_t* d_rank = nullptr;     // {key, idx, n}
    uint8_t* h_stage = nullptr; size_t h_stage_cap = 0;   // pinned landing area of the top-k rows
    uint32_t* h_counts = nullptr;                         // pinned copy of d_counts
    // full sort / filter-only: retained rows
    RowStore ret;
    RowStore in;                    // a post fragment's input, refilled by every sort_feed
};

namespace {

int elem_bytes_of(int prim) { return storage_bytes(prim_storage(prim)); }

void fill_row_args(const SortState* s, const DevCol* cols, int64_t nrows, RowArgs& a) {
    memset(&a, 0, sizeof a);
    for (int i = 0; i < s->ncols; i++) a.cols[i] = cols[i];
    a.n_cols = s->ncols; a.nrows = nrows; a.row_base = s->row_base; a.prog = s->c->prog;
    a.key.pred_out = s->c->ap.pred_out;
    if (!s->c->sort_keys.empty()) {
        const SortKey& k = s->c->sort_keys[0];
        a.key.out_reg = k.out_reg; a.key.vclass = host_prim_class(k.prim); a.key.desc = k.asc ? 0 : 1;
        a.key.direct = s->c->has_direct ? 1 : 0; a.key.col = s->c->has_direct ? s->c->direct_cols[0] : 0;
    }
}

// ---- selection of the k smallest composite keys of one class out of the batch; result merged into the pool ----
int select_topk_class(SortState* s, const RowArgs& ra, int cls, bkgpu_stats* stats) {
    bkgpu_plan* p = s->p;
    const cudaStream_t st = p->stream;
    const int sm_count = p->sm_count;
    Pool& P = s->pool[cls - 1];
    const uint32_t k = (uint32_t)s->k;
    uint32_t* cnt = s->d_counts;     // [0] sample count  [1] level-1 candidates  [2] level-2  [3] rows of this class  [4] kept rows  [5] level-3  [6] two_step: best of the batch
    uint64_t* thr = s->d_rank;       // three {key, idx, n} triples: thresholds of the three levels
    const uint32_t old_n = std::min<uint32_t>(P.n, k);
    // The last level leaves about 1.5 k candidates.  Beside k kept rows they fit one CTA sort only while k is small (at k = 4096 the room
    // would be exactly k: no sampled threshold hits that): a larger k sorts the candidates alone, keeps k, and merges those with the kept rows.
    const bool two_step = old_n > 0 && old_n + 2 * k > SMALL_N;
    const uint32_t room = two_step ? SMALL_N : SMALL_N - old_n;
    const uint32_t trim = std::min<uint32_t>(room, std::max<uint32_t>(2 * k, 2048) - (two_step ? 0 : std::min<uint32_t>(old_n, 1024)));
    const int nxt = P.cur ^ 1;
    const uint64_t* pool_thr = nullptr;
    if (P.n >= k) {   // later rows must beat the k-th composite key kept so far
        CK(p, cudaMemcpyAsync(thr + 12, P.key[P.cur] + (k - 1), 8, cudaMemcpyDeviceToDevice, st));
        CK(p, cudaMemcpyAsync(thr + 13, P.idx[P.cur] + (k - 1), 8, cudaMemcpyDeviceToDevice, st));
        pool_thr = thr + 12;
    }
    uint32_t h[8];
    // The whole chain (sample -> threshold -> compact, three times, then the one-CTA sort and the payload gather)
    // is enqueued without a host round trip; counts are checked once at the end.  A statistically unlucky
    // threshold (too tight / too loose) repeats the chain with wider ranks.
    for (int attempt = 0; attempt < 6; attempt++) {
        const uint32_t widen = 1u << attempt;
        CK(p, cudaMemsetAsync(cnt, 0, 32, st));
        const bool big = ra.nrows > (int64_t)s->cand_cap / 2;
        if (big) {
            k_sample_rows<<<(SAMPLE_N + 255) / 256, 256, 0, st>>>(ra, cls, s->samp_key, s->samp_idx, cnt, 0x5bd1e995ull + attempt * 7919);
            double w = ((double)k * (double)SAMPLE_N / (double)ra.nrows * 1.5 + 32.0) * (double)widen;
            uint32_t rank = w >= (double)(SAMPLE_N - 1) ? 0xFFFFFFFFu : (uint32_t)w;
            k_select_rank<<<1, 1024, 0, st>>>(s->samp_key, s->samp_idx, cnt, SAMPLE_N, rank, thr, nullptr, 0, 0, 0, pool_thr);
            stats->kernel_launches += 2;
        } else if (pool_thr) {
            CK(p, cudaMemcpyAsync(thr, pool_thr, 16, cudaMemcpyDeviceToDevice, st));
        } else CK(p, cudaMemsetAsync(thr, 0xFF, 16, st));
        const DevCol& kc = ra.cols[ra.key.col];
        const bool vec = cls == 1 && ra.key.direct && !kc.validity && (((uintptr_t)kc.values & 31) == 0) && kc.prim != BK_INT8 && kc.prim != BK_INT16 &&
                         kc.prim != BK_UINT8 && kc.prim != BK_UINT16 && (kc.stype == ST_I64 || kc.stype == ST_U64 || kc.stype == ST_F64 || kc.stype == ST_I32 || kc.stype == ST_U32);
        s->used_vec = vec;
        if (vec) {
            const int g = std::max(1, std::min(sm_count * 8, (int)((ra.nrows / 4 + 511) / 512)));
            if (kc.stype == ST_I32 || kc.stype == ST_U32) k_collect_rows_vec<4><<<g, 256, 0, st>>>(ra, thr, s->cand_key[0], s->cand_idx[0], cnt + 1, s->cand_cap, cnt + 3);
            else k_collect_rows_vec<8><<<g, 256, 0, st>>>(ra, thr, s->cand_key[0], s->cand_idx[0], cnt + 1, s->cand_cap, cnt + 3);
        } else
        k_collect_rows<<<grid_for(ra.nrows, sm_count, 8), 256, 0, st>>>(ra, cls, thr, s->cand_key[0], s->cand_idx[0], cnt + 1, s->cand_cap, cnt + 3);
        // level 2: cand[0] (cnt[1]) -> cand[1] (cnt[2]);  level 3: cand[1] (cnt[2]) -> cand[0] (cnt[5])
        const int src_cnt[2] = {1, 2}, dst_cnt[2] = {2, 5};
        for (int lvl = 0; lvl < 2; lvl++) {
            const int from = lvl, to = lvl ^ 1;
            CK(p, cudaMemsetAsync(cnt, 0, 4, st));
            k_sample_pairs<<<(SAMPLE_N + 255) / 256, 256, 0, st>>>(s->cand_key[from], s->cand_idx[from], cnt + src_cnt[lvl], s->cand_cap, s->samp_key, s->samp_idx, cnt,
                                                                   0x9e3779b9ull + attempt * 104729 + lvl);
            // (levels keep trimming until about two k-fulls are left: the one-CTA sort below costs 35 us for <= 2048 keys, 150 us for 8192)
            k_select_rank<<<1, 1024, 0, st>>>(s->samp_key, s->samp_idx, cnt, SAMPLE_N, 0, thr + 3 * (lvl + 1), cnt + src_cnt[lvl], k, widen, trim, nullptr);
            k_collect_pairs<<<grid_for(lvl == 0 ? (int64_t)s->cand_cap / 4 : 65536, sm_count, 8), 256, 0, st>>>(
                s->cand_key[from], s->cand_idx[from], cnt + src_cnt[lvl], thr + 3 * (lvl + 1), s->cand_key[to], s->cand_idx[to], cnt + dst_cnt[lvl], s->cand_cap);
            stats->kernel_launches += 3;
        }
        // final: candidates + kept rows sorted by one CTA, keep k, fetch the payload of the survivors
        if (two_step) {   // cand[0] (cnt[5]) -> its k best in cand[1] (cnt[6]) -> merged with the kept rows
            k_sort_small<<<1, 1024, SMALL_N * 16, st>>>(s->cand_key[0], s->cand_idx[0], cnt + 5, room, nullptr, nullptr, 0,
                                                        s->cand_key[1], s->cand_idx[1], k, cnt + 6, 0, nullptr, nullptr, 0, 0, 0, nullptr);
            k_sort_small<<<1, 1024, SMALL_N * 16, st>>>(s->cand_key[1], s->cand_idx[1], cnt + 6, k, P.key[P.cur], P.idx[P.cur], old_n,
                                                        P.key[nxt], P.idx[nxt], k, cnt + 4, 0, nullptr, nullptr, 0, 0, 0, nullptr);
            stats->kernel_launches++;
        } else
        k_sort_small<<<1, 1024, SMALL_N * 16, st>>>(s->cand_key[0], s->cand_idx[0], cnt + 5, room, P.key[P.cur], P.idx[P.cur], old_n,
                                                    P.key[nxt], P.idx[nxt], k, cnt + 4, 0, nullptr, nullptr, 0, 0, 0, nullptr);
        GatherArgs g; memset(&g, 0, sizeof g);
        for (int i = 0; i < s->ncols; i++) { g.cols[i] = ra.cols[i]; g.dst_vals[i] = P.vals[nxt][i]; g.dst_null[i] = P.nulls[nxt][i]; g.old_vals[i] = P.vals[P.cur][i]; g.old_null[i] = P.nulls[P.cur][i]; }
        g.n_cols = s->ncols; g.row_base = ra.row_base; g.nrows = ra.nrows; g.old_idx = P.idx[P.cur]; g.old_n = old_n;
        k_gather_topk<<<std::max(1, (int)((k + 127) / 128)), 128, 0, st>>>(g, P.idx[nxt], cnt + 4);
        stats->kernel_launches += 3;
        if (!s->h_counts) CK(p, cudaHostAlloc((void**)&s->h_counts, 64, cudaHostAllocDefault));
        CK(p, cudaMemcpyAsync(s->h_counts, cnt, 32, cudaMemcpyDeviceToHost, st));
        if (big && pool_thr) CK(p, cudaMemcpyAsync(s->h_counts + 8, thr + 2, 8, cudaMemcpyDeviceToHost, st));
        CK(p, cudaStreamSynchronize(st));
        memcpy(h, s->h_counts, 32);
        const uint32_t c1 = h[1], c2 = h[2], cls_rows = h[3], c3 = h[5];
        // fewer than k candidates are complete only when the threshold in force was the pool's k-th key (every row at or below it
        // was collected); a tighter SAMPLE threshold may have cut rows that belong between it and the pool's key: widen and retry
        uint64_t thr_info = 0;
        if (big && pool_thr) memcpy(&thr_info, s->h_counts + 8, 8);
        const bool pool_in_force = pool_thr != nullptr && (!big || ((thr_info >> 62) & 1ull));
        const bool ok1 = c1 <= s->cand_cap && (c1 >= k || c1 >= cls_rows || pool_in_force);
        const bool ok2 = c2 <= s->cand_cap && (c2 >= std::min(k, c1));
        const bool ok3 = c3 <= room && (c3 >= std::min(k, c2));
        if (ok1 && ok2 && ok3) { P.cur = nxt; P.n = h[4]; return 0; }
    }
    return p->fail(BKGPU_ETOOBIG, "top-k selection did not converge (candidate buffers too small for this key distribution)");
}

// rows that pass the predicate are appended, in input order, to the retained columns (filter-only and full sort)
int retain_batch(SortState* s, const RowArgs& ra, bkgpu_stats* stats) {
    const int64_t limit_left = (s->c->kind == PK_FILTER && s->c->limit >= 0) ? std::max<int64_t>(s->c->limit - s->ret.rows, 0) : INT64_MAX;
    if (limit_left == 0) return 0;   // FilterNode stops after `limit` passing rows (filter_node.cpp:786-791)
    bkgpu_plan* p = s->p;
    const cudaStream_t st = p->stream;
    const int64_t rows_per_block = 4096;
    const uint32_t nblocks = (uint32_t)((ra.nrows + rows_per_block - 1) / rows_per_block);
    // counts[b]: the passing rows of block b, scanned into its first output position; counts[nblocks] closes the scan with the total
    DevScope scope(p);
    uint32_t *counts = nullptr, *sums = nullptr, *sel = nullptr; int rc;
    if ((rc = scope.alloc(&counts, ((size_t)nblocks + 1) * 4))) return rc;
    if ((rc = scope.alloc(&sums, (size_t)scan_scratch((int64_t)nblocks + 1) * 4))) return rc;
    CK(p, cudaMemsetAsync(counts + nblocks, 0, 4, st));
    k_filter_count<<<nblocks, 256, 0, st>>>(ra, counts, rows_per_block);
    CK(p, scan_excl(counts, (int64_t)nblocks + 1, sums, p->sm_count, st));
    uint32_t total = 0;
    CK(p, cudaMemcpyAsync(&total, counts + nblocks, 4, cudaMemcpyDeviceToHost, st));
    CK(p, cudaStreamSynchronize(st));
    const uint64_t take = std::min<uint64_t>(total, (uint64_t)limit_left);
    if (take > 0) {
        if ((rc = scope.alloc(&sel, (size_t)take * 4))) return rc;
        k_filter_write<<<nblocks, 256, 0, st>>>(ra, counts, rows_per_block, sel, 0, take);
        if ((rc = store_retain(p, s->ret, s->ret.rows + (int64_t)take))) return rc;
        GatherArgs g; memset(&g, 0, sizeof g);
        for (int i = 0; i < s->ncols; i++) { g.cols[i] = ra.cols[i]; g.dst_vals[i] = s->ret.cols[(size_t)i].vals; g.dst_null[i] = s->ret.cols[(size_t)i].nulls; }
        g.n_cols = s->ncols;
        k_gather_sel<<<grid_for((int64_t)take, p->sm_count, 8), 256, 0, st>>>(g, sel, take, (uint64_t)s->ret.rows);
        CK(p, cudaStreamSynchronize(st));
        s->ret.rows += (int64_t)take;
        stats->kernel_launches += 2;
    }
    stats->kernel_launches += 2;   // the count and the scan: one launch up to 2048 blocks (8M rows), three beyond
    stats->rows_filtered += ra.nrows - (int64_t)total;
    return 0;
}

// the buffers of one radix sort of n (key image, row id) pairs, returned to the plan's allocator when it leaves scope
struct RadixBufs {
    DevScope scope;
    uint64_t *img_row = nullptr, *img[2] = {nullptr, nullptr}; uint32_t* ids[2] = {nullptr, nullptr};
    RadixScratch scratch;   // radix_sort's, grown as its sorts need
    uint32_t n = 0;
    explicit RadixBufs(bkgpu_plan* p) : scope(p) {}
    ~RadixBufs() { dev_free(scope.p, scratch.hist); dev_free(scope.p, scratch.status); }
    int alloc(int64_t rows) {
        n = (uint32_t)rows;
        int rc;
        if ((rc = scope.alloc(&img_row, (size_t)n * 8)) || (rc = scope.alloc(&img[0], (size_t)n * 8)) || (rc = scope.alloc(&img[1], (size_t)n * 8)) ||
            (rc = scope.alloc(&ids[0], (size_t)n * 4)) || (rc = scope.alloc(&ids[1], (size_t)n * 4)))
            return rc;
        return 0;
    }
};

// stable LSD radix sort of the row ids b.ids[cur] by `keys` (least significant first).  Key k's image comes from program progs[k] (its
// output register keys[k].out_reg), or straight from column `direct_col` when that is >= 0 (one key).  identity_start: b.ids[cur] holds
// 0..n-1, so the first key's images need no gather into the current order.
int radix_sort_keys(SortState* s, RowArgs& ra, const std::vector<SortKey>& keys, const std::vector<const Program*>& progs, int direct_col,
                    bool direct_has_nulls, RadixBufs& b, int& cur, bool identity_start, bkgpu_stats* stats, int64_t& pass_bytes) {
    bkgpu_plan* p = s->p;
    const cudaStream_t st = p->stream;
    const int sm = p->sm_count;
    const int64_t n = b.n;
    uint64_t** img = b.img; uint32_t** ids = b.ids; uint64_t* img_row = b.img_row;
    bool first = identity_start;
    for (int ki = (int)keys.size() - 1; ki >= 0; ki--) {
        const SortKey& sk = keys[(size_t)ki];
        ra.prog = *progs[(size_t)ki];
        for (int mode = 0; mode < 2; mode++) {   // the key's value image first, then its NULL rank (stable: NULLs end up strictly first / last)
            if (mode == 1 && direct_col >= 0 && !direct_has_nulls) continue;
            uint64_t* dst = first ? img[cur] : img_row;
            if (mode == 0 && direct_col >= 0) k_sort_images_direct<<<grid_for(n, sm, 8), 256, 0, st>>>(ra.cols[direct_col], n, host_prim_class(sk.prim), sk.asc ? 0 : 1, dst);
            else
            k_sort_images<<<grid_for(n, sm, 8), 256, 0, st>>>(ra, sk.out_reg, host_prim_class(sk.prim), sk.asc ? 0 : 1, sk.null_first ? 1 : 0, mode, dst, nullptr);
            if (!first) k_rs_gather_u64<<<grid_for(n, sm, 8), 256, 0, st>>>(img_row, ids[cur], img[cur], b.n);   // images in the current order
            first = false;
            stats->kernel_launches += 2;
            const int r = radix_sort(p, img, ids, cur, n, b.scratch, stats, &pass_bytes);
            if (r < 0) return r;
            cur = r;
        }
    }
    return 0;
}
}  // namespace

// ------------------------------------------------------------------------------------------------------------
int sort_open(bkgpu_plan* p, const Compiled& c, int64_t region_base, SortState** out) {
    SortState* s = new SortState();
    s->p = p; s->c = &c; s->ncols = (int)c.cols.size();
    s->row_base = s->region_base = (uint64_t)region_base;
    s->k = c.kind == PK_SORT ? c.limit : -1;
    s->topk = c.kind == PK_SORT && c.sort_keys.size() == 1 && s->k >= 0 && s->k <= 4096;
    store_init(s->ret, c.cols);
    store_init(s->in, c.cols);
    int rc = 0;
    if (s->topk) {
        s->cand_cap = 1u << 22;   // 4M candidate pairs (64 MB per array pair)
        const size_t kk = (size_t)std::max<int64_t>(s->k, 1);
        for (int b = 0; b < 2 && !rc; b++) {
            if ((rc = dev_alloc(p, (void**)&s->cand_key[b], (size_t)s->cand_cap * 8))) break;
            if ((rc = dev_alloc(p, (void**)&s->cand_idx[b], (size_t)s->cand_cap * 8))) break;
        }
        if (!rc) rc = dev_alloc(p, (void**)&s->samp_key, SAMPLE_N * 8);
        if (!rc) rc = dev_alloc(p, (void**)&s->samp_idx, SAMPLE_N * 8);
        if (!rc) rc = dev_alloc(p, (void**)&s->d_counts, 64);
        if (!rc) rc = dev_alloc(p, (void**)&s->d_rank, 128);
        for (int q = 0; q < 2 && !rc; q++) for (int b = 0; b < 2 && !rc; b++) {
            if ((rc = dev_alloc(p, (void**)&s->pool[q].key[b], kk * 8))) break;
            if ((rc = dev_alloc(p, (void**)&s->pool[q].idx[b], kk * 8))) break;
            for (int ci = 0; ci < s->ncols && !rc; ci++) {
                if ((rc = dev_alloc(p, (void**)&s->pool[q].vals[b][ci], kk * (size_t)elem_bytes_of(c.cols[(size_t)ci].prim)))) break;
                rc = dev_alloc(p, (void**)&s->pool[q].nulls[b][ci], kk);
            }
        }
        if (!rc) { cudaError_t e = cudaFuncSetAttribute(k_sort_small, cudaFuncAttributeMaxDynamicSharedMemorySize, SMALL_N * 16); if (e != cudaSuccess) rc = p->cuda_fail(e, "cudaFuncSetAttribute"); }
    }
    if (rc) { sort_close(s); return rc; }
    *out = s;
    return 0;
}

void sort_reset(SortState* s) {
    for (auto& P : s->pool) { P.n = 0; P.cur = 0; }
    s->ret.rows = 0;
    s->row_base = s->region_base;
}

int sort_push(SortState* s, const DevCol* cols, int64_t nrows, bkgpu_stats* stats) {
    if (nrows > 0x7FFFFFFFll) return s->p->fail(BKGPU_EUNSUPPORTED, "a single pushed batch of a SORT/FILTER plan is limited to 2^31-1 rows");
    const cudaStream_t stream = s->p->stream;
    RowArgs ra; fill_row_args(s, cols, nrows, ra);
    int rc = 0;
    if (s->topk) {
        if (s->k == 0) { s->row_base += (uint64_t)nrows; return 0; }
        StageTimer t;
        cudaEventRecord(t.a, stream);
        rc = select_topk_class(s, ra, 1, stats);
        const bool need_nulls = ra.key.direct ? cols[ra.key.col].validity != nullptr : true;
        if (!rc && need_nulls) rc = select_topk_class(s, ra, 2, stats);
        cudaEventRecord(t.b, stream); cudaEventSynchronize(t.b);
        float ms = 0; cudaEventElapsedTime(&ms, t.a, t.b);
        stats->main_kernel_ms += ms; stats->main_kernel_launches += 1;
        stats->main_kernel_bytes += nrows * (ra.key.direct ? storage_bytes(cols[ra.key.col].stype) : 8);
        snprintf(stats->main_kernel_name, sizeof stats->main_kernel_name, "%s", s->used_vec ? "topk_select(k_collect_rows_vec)" : "topk_select(k_collect_rows)");
    } else {
        rc = retain_batch(s, ra, stats);
        snprintf(stats->main_kernel_name, sizeof stats->main_kernel_name, "%s", s->c->kind == PK_FILTER ? "k_filter_write" : "radix_sort(k_rs_pass)");
    }
    s->row_base += (uint64_t)nrows;
    return rc;
}

int sort_feed(SortState* s, int64_t n, int64_t cap, int per_sm, bkgpu_stats* stats, const std::function<int(RowStore& in)>& fill) {
    if (n == 0) return BKGPU_OK;
    bkgpu_plan* p = s->p;
    int rc;
    for (size_t k = 0; k < s->in.cols.size(); k++)
        if ((rc = store_reserve(p, s->in, k, n, cap, true))) return rc;
    if ((rc = fill(s->in))) return rc;
    std::vector<DevCol> dc(std::max<size_t>(s->in.cols.size(), 1));
    for (size_t k = 0; k < s->in.cols.size(); k++)
        if ((rc = store_pack(p, s->in, k, n, per_sm, nullptr, &dc[k]))) return rc;
    return sort_push(s, dc.data(), n, stats);
}

// layout of the exported partial (top-k): [u64 n][k keys][k idx][per column: k values (8-byte slots)][per column: k null bytes padded to 8]
size_t sort_partial_bytes(SortState* s) {
    if (!s->topk) return 0;
    const size_t k = (size_t)std::max<int64_t>(s->k, 1);
    return 8 * (1 + 2 * 2 * k) + (size_t)s->ncols * 2 * (k * 8 + ((k + 7) & ~(size_t)7));
}

// host image of the k best rows of this rank: class-tagged, ready to be merged with other ranks'
struct HostRows {
    std::vector<uint8_t> cls; std::vector<uint64_t> key, idx;
    std::vector<std::vector<uint8_t>> vals, nulls;   // per column, row-major fixed width
};

// the k surviving rows of both pools (keys present / NULL keys) land in ONE pinned staging block: every copy is truly
// asynchronous and the whole result costs a single synchronisation
static int topk_host_rows(SortState* s, HostRows& h) {
    bkgpu_plan* p = s->p;
    const cudaStream_t st = p->stream;
    h.vals.assign((size_t)s->ncols, {}); h.nulls.assign((size_t)s->ncols, {});
    size_t row_bytes = 16;
    for (int c = 0; c < s->ncols; c++) row_bytes += (size_t)elem_bytes_of(s->c->cols[(size_t)c].prim) + 1;
    const size_t n_tot = (size_t)s->pool[0].n + (size_t)s->pool[1].n;
    const size_t need = n_tot * row_bytes + 64 * (size_t)(s->ncols + 2) * 2;
    if (s->h_stage_cap < need) {
        if (s->h_stage) cudaFreeHost(s->h_stage);
        s->h_stage = nullptr; s->h_stage_cap = 0;
        CK(p, cudaHostAlloc((void**)&s->h_stage, need * 2, cudaHostAllocDefault));
        s->h_stage_cap = need * 2;
    }
    struct Seg { size_t key, idx; std::vector<size_t> val, nul; } seg[2];
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 63) & ~(size_t)63; return o; };
    for (int q = 0; q < 2; q++) {
        Pool& P = s->pool[q];
        const size_t n = P.n;
        if (!n) continue;
        seg[q].key = take(n * 8); seg[q].idx = take(n * 8);
        CK(p, cudaMemcpyAsync(s->h_stage + seg[q].key, P.key[P.cur], n * 8, cudaMemcpyDeviceToHost, st));
        CK(p, cudaMemcpyAsync(s->h_stage + seg[q].idx, P.idx[P.cur], n * 8, cudaMemcpyDeviceToHost, st));
        for (int c = 0; c < s->ncols; c++) {
            const size_t eb = (size_t)elem_bytes_of(s->c->cols[(size_t)c].prim);
            seg[q].val.push_back(take(n * eb)); seg[q].nul.push_back(take(n));
            CK(p, cudaMemcpyAsync(s->h_stage + seg[q].val.back(), P.vals[P.cur][c], n * eb, cudaMemcpyDeviceToHost, st));
            CK(p, cudaMemcpyAsync(s->h_stage + seg[q].nul.back(), P.nulls[P.cur][c], n, cudaMemcpyDeviceToHost, st));
        }
    }
    CK(p, cudaStreamSynchronize(st));
    for (int q = 0; q < 2; q++) {
        const size_t n = s->pool[q].n;
        if (!n) continue;
        const uint64_t* key = (const uint64_t*)(s->h_stage + seg[q].key); const uint64_t* idx = (const uint64_t*)(s->h_stage + seg[q].idx);
        for (size_t i = 0; i < n; i++) { h.cls.push_back((uint8_t)(q + 1)); h.key.push_back(key[i]); h.idx.push_back(idx[i]); }
        for (int c = 0; c < s->ncols; c++) {
            const size_t eb = (size_t)elem_bytes_of(s->c->cols[(size_t)c].prim);
            const uint8_t* v = s->h_stage + seg[q].val[(size_t)c]; const uint8_t* nb = s->h_stage + seg[q].nul[(size_t)c];
            h.vals[(size_t)c].insert(h.vals[(size_t)c].end(), v, v + n * eb);
            h.nulls[(size_t)c].insert(h.nulls[(size_t)c].end(), nb, nb + n);
        }
    }
    return 0;
}
// the first k rows of h in ORDER BY order, after OFFSET, into p->result
static void finish_host_rows(SortState* s, const HostRows& h) {
    const bool null_first = s->c->sort_keys[0].null_first;
    std::vector<uint32_t> order(h.key.size());
    for (size_t i = 0; i < order.size(); i++) order[i] = (uint32_t)i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
        const int ra = h.cls[a] == 2 ? (null_first ? 0 : 2) : 1, rb = h.cls[b] == 2 ? (null_first ? 0 : 2) : 1;
        if (ra != rb) return ra < rb;
        if (h.key[a] != h.key[b]) return h.key[a] < h.key[b];
        return h.idx[a] < h.idx[b];
    });
    int64_t n = (int64_t)order.size();
    if (s->k >= 0 && n > s->k) n = s->k;
    int64_t skip = std::min<int64_t>(s->c->offset, n);
    n -= skip;
    bkgpu_plan* p = s->p;
    p->result.clear();
    for (int c = 0; c < s->ncols; c++) {
        const ColRef& cr = s->c->cols[(size_t)c];
        HostCol oc; oc.desc = OutCol{cr.tuple_id, cr.slot_id, cr.prim, 0}; oc.elem = elem_bytes_of(cr.prim);
        oc.values.assign((size_t)std::max<int64_t>(n, 1) * oc.elem, 0);
        bool any = false;
        std::vector<uint8_t> valid((size_t)(n + 7) / 8 + 1, 0xFF);
        for (int64_t i = 0; i < n; i++) {
            const uint32_t src = order[(size_t)(i + skip)];
            memcpy(oc.values.data() + (size_t)i * oc.elem, h.vals[(size_t)c].data() + (size_t)src * oc.elem, (size_t)oc.elem);
            if (h.nulls[(size_t)c][src]) { any = true; valid[(size_t)i >> 3] &= (uint8_t)~(1u << (i & 7)); }
        }
        if (any) oc.validity = std::move(valid);
        p->result.push_back(std::move(oc));
    }
    p->result_rows = n; p->result_pos = 0;
}

static void pack_rows(SortState* s, const HostRows& h, std::vector<uint64_t>& buf) {
    const size_t k = (size_t)std::max<int64_t>(s->k, 1), kk = 2 * k;   // both classes
    const size_t nullw = (k + 7) / 8;
    buf.assign(sort_partial_bytes(s) / 8, 0);
    const size_t n = std::min(h.key.size(), kk);
    buf[0] = n;
    uint64_t* keys = buf.data() + 1; uint64_t* idx = keys + kk;
    uint64_t* col0 = idx + kk;
    for (size_t i = 0; i < n; i++) { keys[i] = h.key[i]; idx[i] = h.idx[i] | ((uint64_t)(h.cls[i] == 2) << 63); }
    for (int c = 0; c < s->ncols; c++) {
        const int eb = elem_bytes_of(s->c->cols[(size_t)c].prim);
        uint64_t* v = col0 + (size_t)c * 2 * (k + nullw);
        uint8_t* nb = (uint8_t*)(v + kk);
        for (size_t i = 0; i < n; i++) { memcpy(&v[i], h.vals[(size_t)c].data() + i * eb, (size_t)eb); nb[i] = h.nulls[(size_t)c][i]; }
    }
}
static void unpack_rows(SortState* s, const uint64_t* buf, HostRows& h) {
    const size_t k = (size_t)std::max<int64_t>(s->k, 1), kk = 2 * k, nullw = (k + 7) / 8;
    const size_t n = (size_t)buf[0];
    const uint64_t* keys = buf + 1; const uint64_t* idx = keys + kk; const uint64_t* col0 = idx + kk;
    if (h.vals.empty()) { h.vals.assign((size_t)s->ncols, {}); h.nulls.assign((size_t)s->ncols, {}); }
    for (size_t i = 0; i < n; i++) { h.key.push_back(keys[i]); h.idx.push_back(idx[i] & ~(1ull << 63)); h.cls.push_back((idx[i] >> 63) ? 2 : 1); }
    for (int c = 0; c < s->ncols; c++) {
        const int eb = elem_bytes_of(s->c->cols[(size_t)c].prim);
        const uint64_t* v = col0 + (size_t)c * 2 * (k + nullw);
        const uint8_t* nb = (const uint8_t*)(v + kk);
        for (size_t i = 0; i < n; i++) {
            const uint8_t* p = (const uint8_t*)&v[i];
            h.vals[(size_t)c].insert(h.vals[(size_t)c].end(), p, p + eb);
            h.nulls[(size_t)c].push_back(nb[i]);
        }
    }
}

int sort_partial_export(SortState* s, void* dev_dst) {
    bkgpu_plan* p = s->p;
    if (!s->topk) return p->fail(BKGPU_EUNSUPPORTED, "only ORDER BY ... LIMIT plans have a partial state");
    HostRows h; int rc = topk_host_rows(s, h);
    if (rc) return rc;
    std::vector<uint64_t> buf; pack_rows(s, h, buf);
    CK(p, cudaMemcpyAsync(dev_dst, buf.data(), buf.size() * 8, cudaMemcpyHostToDevice, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    return 0;
}

int sort_partial_merge(SortState* s, const void* dev_src, int nranks) {
    bkgpu_plan* p = s->p;
    if (!s->topk) return p->fail(BKGPU_EUNSUPPORTED, "only ORDER BY ... LIMIT plans have a partial state");
    const size_t words = sort_partial_bytes(s) / 8;
    std::vector<uint64_t> all(words * (size_t)nranks);
    CK(p, cudaMemcpyAsync(all.data(), dev_src, all.size() * 8, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    HostRows h;
    for (int r = 0; r < nranks; r++) unpack_rows(s, all.data() + (size_t)r * words, h);
    finish_host_rows(s, h);   // SelectManagerNode's merge of per-region sorted runs (select_manager_node.cpp:50-51)
    return 0;
}

static int finish_rows(SortState* s, void* nccl_comm, int nranks, bkgpu_stats* stats) {
    bkgpu_plan* p = s->p;
    const cudaStream_t st = p->stream;
    if (s->topk) {
        HostRows h; int rc = topk_host_rows(s, h);
        if (rc) return rc;
        if (nccl_comm && nranks > 1) {   // per-GPU top-k rows meet in one all-gather; every rank finishes the merge
            std::vector<uint64_t> buf; pack_rows(s, h, buf);
            DevScope scope(p);
            uint64_t *d_send = nullptr, *d_recv = nullptr;
            if ((rc = scope.alloc(&d_send, buf.size() * 8))) return rc;
            if ((rc = scope.alloc(&d_recv, buf.size() * 8 * (size_t)nranks))) return rc;
            StageTimer t;
            CK(p, cudaMemcpyAsync(d_send, buf.data(), buf.size() * 8, cudaMemcpyHostToDevice, st));
            cudaEventRecord(t.a, st);
            if (nccl_all_gather(nccl_comm, d_send, d_recv, buf.size(), st) != 0) return p->fail(BKGPU_ENCCL, "ncclAllGather: %s", nccl_last_error());
            cudaEventRecord(t.b, st);
            rc = sort_partial_merge(s, d_recv, nranks);
            float ms = 0; cudaEventElapsedTime(&ms, t.a, t.b); stats->collective_ms += ms;
            return rc;
        }
        finish_host_rows(s, h);
        return 0;
    }
    if (nccl_comm && nranks > 1) return p->fail(BKGPU_EUNSUPPORTED, "multi-GPU merge is implemented for ORDER BY ... LIMIT (top-k) and aggregates");
    if (s->c->kind == PK_FILTER) {
        int64_t n = s->ret.rows;
        int64_t skip = std::min<int64_t>(s->c->offset, n);
        n -= skip;
        return store_copy_out(p, s->ret, s->c->cols, nullptr, n, skip);
    }
    // ---- full ORDER BY: stable LSD radix sort of (key image, row id) pairs, least significant ORDER BY key first ----
    const int64_t n = s->ret.rows;
    if (n > RADIX_MAX_KEYS) return p->fail(BKGPU_EUNSUPPORTED, "full sort is limited to 2^30 - 1 rows per GPU");
    if (n == 0) return store_copy_out(p, s->ret, s->c->cols, nullptr, 0, 0);
    RadixBufs b(p); int rc;
    if ((rc = b.alloc(n))) return rc;
    RowArgs ra; memset(&ra, 0, sizeof ra);
    // retained columns carry null BYTES: pack them into bitmaps on the device so the key program sees NULLs; h_null_flags[c]: column c
    // holds a NULL
    uint32_t h_null_flags[MAX_COLS] = {0};
    {
        DevScope flags_scope(p);
        uint32_t* null_flags = nullptr;
        if ((rc = flags_scope.alloc(&null_flags, sizeof(uint32_t) * MAX_COLS))) return rc;
        CK(p, cudaMemsetAsync(null_flags, 0, sizeof(uint32_t) * MAX_COLS, st));
        for (int c = 0; c < s->ncols; c++)
            if ((rc = store_pack(p, s->ret, (size_t)c, n, 8, null_flags + c, &ra.cols[c]))) return rc;
        CK(p, cudaMemcpyAsync(h_null_flags, null_flags, sizeof(uint32_t) * (size_t)s->ncols, cudaMemcpyDeviceToHost, st));
        CK(p, cudaStreamSynchronize(st));
    }
    ra.n_cols = s->ncols; ra.nrows = n; ra.prog = s->c->prog; ra.key.pred_out = -1;
    k_iota<<<grid_for(n, p->sm_count, 8), 256, 0, st>>>(b.ids[0], n);
    int cur = 0;
    StageTimer t;
    cudaEventRecord(t.a, st);
    int64_t pass_bytes = 0;
    // a plain column key (config C5's shape): its image comes straight from the column, and without NULLs in it the NULL-rank pass is void
    const bool direct_key = s->c->has_direct && s->c->sort_keys.size() == 1 && !s->c->direct_cols.empty();
    const int dcol = direct_key ? s->c->direct_cols[0] : -1;
    std::vector<const Program*> progs(s->c->sort_keys.size(), &s->c->prog);
    if ((rc = radix_sort_keys(s, ra, s->c->sort_keys, progs, dcol, dcol >= 0 && h_null_flags[dcol], b, cur, true, stats, pass_bytes))) return rc;
    cudaEventRecord(t.b, st);
    CK(p, cudaStreamSynchronize(st));
    { float ms = 0; cudaEventElapsedTime(&ms, t.a, t.b); stats->main_kernel_ms += ms; stats->main_kernel_launches += 1; stats->main_kernel_bytes += pass_bytes; }
    snprintf(stats->main_kernel_name, sizeof stats->main_kernel_name, "%s", "radix_sort(k_rs_pass)");
    int64_t keep = n; if (s->k >= 0 && keep > s->k) keep = s->k;
    int64_t skip = std::min<int64_t>(s->c->offset, keep); keep -= skip;
    return store_copy_out(p, s->ret, s->c->cols, b.ids[cur], keep, skip);
}

int sort_finish(SortState* s, void* nccl_comm, int nranks, bkgpu_stats* stats, const OutCol* desc) {
    const int rc = finish_rows(s, nccl_comm, nranks, stats);
    if (!rc && desc) for (size_t k = 0; k < s->p->result.size(); k++) s->p->result[k].desc = desc[k];
    return rc;
}

// ---- the window stage's access to the retained rows and the radix sort (window.cu) ----
RowStore& sort_retained(SortState* s) { return s->ret; }

int sort_stable_ids(SortState* s, const DevCol* cols, int64_t n, const std::vector<SortKey>& keys, const std::vector<const Program*>& progs,
                    uint32_t* ids, bkgpu_stats* stats) {
    if (n == 0 || keys.empty()) return 0;
    bkgpu_plan* p = s->p;
    RadixBufs b(p); int rc;
    if ((rc = b.alloc(n))) return rc;
    RowArgs ra; memset(&ra, 0, sizeof ra);
    for (int c = 0; c < s->ncols; c++) ra.cols[c] = cols[c];
    ra.n_cols = s->ncols; ra.nrows = n; ra.key.pred_out = -1;
    CK(p, cudaMemcpyAsync(b.ids[0], ids, (size_t)n * 4, cudaMemcpyDeviceToDevice, p->stream));
    int cur = 0; int64_t pass_bytes = 0;
    if ((rc = radix_sort_keys(s, ra, keys, progs, -1, true, b, cur, false, stats, pass_bytes))) return rc;
    CK(p, cudaMemcpyAsync(ids, b.ids[cur], (size_t)n * 4, cudaMemcpyDeviceToDevice, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    return 0;
}

// (the device buffers belong to the plan: bkgpu_close returns them)
void sort_close(SortState* s) {
    if (!s) return;
    if (s->h_stage) cudaFreeHost(s->h_stage);
    if (s->h_counts) cudaFreeHost(s->h_counts);
    delete s;
}

}  // namespace bk

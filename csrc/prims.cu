// prims.cu — device primitives shared by ORDER BY and the window stage (sort.cu, window.cu), the hash join (join.cu) and rb_build_agg
// (rb.cu), for sm_90a.
#include "prims.cuh"
#include <string.h>
#include <algorithm>
#include "api_state.h"
#include "dev_common.cuh"

namespace bk {

int grid_for(int64_t n, int sm, int per_sm) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sm * per_sm)); }

__global__ void k_iota(uint32_t* ids, int64_t n) { for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) ids[i] = (uint32_t)i; }

__global__ void k_pack_null_bytes(const uint8_t* nb, int64_t n, uint8_t* bitmap, uint32_t* any_null) {
    const int64_t nbytes = (n + 7) / 8;
    bool seen = false;
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nbytes; b += (int64_t)gridDim.x * blockDim.x) {
        uint32_t v = 0;
        for (int j = 0; j < 8; j++) { const int64_t r = b * 8 + j; if (r < n) { if (!nb[r]) v |= 1u << j; else seen = true; } }
        bitmap[b] = (uint8_t)v;
    }
    if (seen && any_null) *any_null = 1u;   // (lets the sort skip the NULL-rank pass of a key column without NULLs)
}

// Arrow validity bitmap (nullptr: every row valid) -> null BYTES
__global__ void k_unpack_validity(const uint8_t* bitmap, int64_t n, uint8_t* null_bytes) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        null_bytes[i] = bitmap ? (((bitmap[i >> 3] >> (i & 7)) & 1) ? 0 : 1) : 0;
}

__global__ void k_gather_sel(GatherArgs g, const uint32_t* sel, uint64_t n, uint64_t dst_off) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const int64_t src = sel[i];
        for (int c = 0; c < g.n_cols; c++) {
            const int eb = g.cols[c].stype == ST_U8 ? 1 : (g.cols[c].stype == ST_BLOB16 ? 16 : ((g.cols[c].stype == ST_I32 || g.cols[c].stype == ST_U32 || g.cols[c].stype == ST_F32) ? 4 : 8));
            const uint8_t* sv = (const uint8_t*)g.cols[c].values + (size_t)src * eb;
            uint8_t* dv = g.dst_vals[c] + (size_t)(dst_off + i) * eb;
            if (eb == 8) *(uint64_t*)dv = *(const uint64_t*)sv; else if (eb == 4) *(uint32_t*)dv = *(const uint32_t*)sv;
            else if (eb == 16) { ((uint64_t*)dv)[0] = ((const uint64_t*)sv)[0]; ((uint64_t*)dv)[1] = ((const uint64_t*)sv)[1]; }   // AVG intermediate blob (payload only)
            else *dv = *sv;
            g.dst_null[c][dst_off + i] = elem_is_null(g.cols[c], src) ? 1 : 0;
        }
    }
}

namespace {

__global__ void k_rs_gather_bytes(const uint8_t* src, const uint32_t* ids, uint8_t* dst, uint64_t n) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) dst[i] = src[ids[i]];
}

int elem_bytes_of(int prim) { return storage_bytes(prim_storage(prim)); }

// *buf reallocated with `bytes`, its first `keep` bytes copied over
int regrow(bkgpu_plan* p, uint8_t** buf, size_t bytes, size_t keep) {
    uint8_t* nb = nullptr;
    int rc;
    if ((rc = dev_alloc(p, (void**)&nb, bytes))) return rc;
    if (keep) {
        CK(p, cudaMemcpyAsync(nb, *buf, keep, cudaMemcpyDeviceToDevice, p->stream));
        CK(p, cudaStreamSynchronize(p->stream));
    }
    dev_free(p, *buf);
    *buf = nb;
    return BKGPU_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------
void store_init(RowStore& s, const std::vector<ColRef>& cols) {
    s.cols.assign(cols.size(), RowStore::Col{});
    for (size_t i = 0; i < cols.size(); i++) s.cols[i].prim = cols[i].prim;
}

int store_reserve(bkgpu_plan* p, RowStore& s, size_t i, int64_t need, int64_t cap, bool nulls) {
    RowStore::Col& c = s.cols[i];
    const size_t eb = (size_t)elem_bytes_of(c.prim);
    int rc;
    if (c.cap < need) {
        if ((rc = regrow(p, &c.vals, (size_t)cap * eb + 64, (size_t)s.rows * eb))) return rc;
        c.cap = cap;
    }
    if (nulls && c.null_cap < need) {
        if ((rc = regrow(p, &c.nulls, (size_t)cap + 64, (size_t)s.rows)) || (rc = regrow(p, &c.bitmap, (size_t)(cap + 7) / 8 + 64, 0))) return rc;
        c.null_cap = cap;
    }
    return BKGPU_OK;
}

int store_retain(bkgpu_plan* p, RowStore& s, int64_t need) {
    if (need <= s.cap) return BKGPU_OK;
    const int64_t cap = std::max<int64_t>(need, std::max<int64_t>(s.cap * 2, 1 << 16));
    int rc;
    for (size_t i = 0; i < s.cols.size(); i++)
        if (s.cols[i].prim >= 0 && (rc = store_reserve(p, s, i, need, cap, true))) return rc;
    s.cap = cap;
    return BKGPU_OK;
}

int store_append(bkgpu_plan* p, RowStore& s, size_t i, const bkgpu_column& in, int64_t n, bool on_device) {
    RowStore::Col& c = s.cols[i];
    const size_t eb = (size_t)elem_bytes_of(c.prim);
    uint8_t* dv = c.vals + (size_t)s.rows * eb;
    uint8_t* dn = c.nulls + s.rows;
    if (on_device) {
        CK(p, cudaMemcpyAsync(dv, in.values, (size_t)n * eb, cudaMemcpyDeviceToDevice, p->stream));
        if (n > 0) k_unpack_validity<<<grid_for(n, p->sm_count, 16), 256, 0, p->stream>>>(in.validity, n, dn);
        CK(p, cudaGetLastError());
    } else {
        CK(p, cudaMemcpyAsync(dv, in.values, (size_t)n * eb, cudaMemcpyHostToDevice, p->stream));
        std::vector<uint8_t> nb((size_t)n, 0);
        if (in.validity) for (int64_t r = 0; r < n; r++) nb[(size_t)r] = ((in.validity[r >> 3] >> (r & 7)) & 1) ? 0 : 1;
        CK(p, cudaMemcpyAsync(dn, nb.data(), (size_t)n, cudaMemcpyHostToDevice, p->stream));
        CK(p, cudaStreamSynchronize(p->stream));
        p->stats.h2d_bytes += (int64_t)((size_t)n * (eb + 1));
    }
    if (in.validity) c.nullable = true;
    return BKGPU_OK;
}

int store_pack(bkgpu_plan* p, const RowStore& s, size_t i, int64_t n, int per_sm, uint32_t* any_null, DevCol* out) {
    const RowStore::Col& c = s.cols[i];
    if (n > 0) k_pack_null_bytes<<<grid_for((n + 7) / 8, p->sm_count, per_sm), 256, 0, p->stream>>>(c.nulls, n, c.bitmap, any_null);
    CK(p, cudaGetLastError());
    *out = store_col(s, i);
    out->validity = c.bitmap;
    return BKGPU_OK;
}

DevCol store_col(const RowStore& s, size_t i) {
    const RowStore::Col& c = s.cols[i];
    DevCol d{};
    d.values = c.vals; d.validity = c.nullable ? c.bitmap : nullptr; d.stype = prim_storage(c.prim); d.prim = c.prim;
    return d;
}

int store_gather(bkgpu_plan* p, const RowStore::Col& src, const uint32_t* perm, int64_t n, uint8_t* dst_vals, uint8_t* dst_nulls) {
    if (n <= 0) return BKGPU_OK;
    const cudaStream_t st = p->stream;
    GatherArgs g; memset(&g, 0, sizeof g);
    g.cols[0].values = src.vals; g.cols[0].validity = nullptr; g.cols[0].stype = prim_storage(src.prim); g.cols[0].prim = src.prim;
    g.n_cols = 1; g.dst_vals[0] = dst_vals; g.dst_null[0] = dst_nulls;
    k_gather_sel<<<grid_for(n, p->sm_count, 8), 256, 0, st>>>(g, perm, (uint64_t)n, 0);
    // null bytes travel separately (k_gather_sel reads validity bitmaps)
    k_rs_gather_bytes<<<grid_for(n, p->sm_count, 8), 256, 0, st>>>(src.nulls, perm, dst_nulls, (uint64_t)n);
    CK(p, cudaGetLastError());
    return BKGPU_OK;
}

int store_copy_out(bkgpu_plan* p, const RowStore& s, const std::vector<ColRef>& desc, const uint32_t* perm, int64_t n, int64_t skip) {
    const cudaStream_t st = p->stream;
    p->result.clear();
    for (size_t c = 0; c < desc.size(); c++) {
        const ColRef& cr = desc[c];
        HostCol oc; oc.desc = OutCol{cr.tuple_id, cr.slot_id, cr.prim, 0}; oc.elem = elem_bytes_of(cr.prim);
        oc.values.assign((size_t)std::max<int64_t>(n, 1) * oc.elem, 0);
        std::vector<uint8_t> nb((size_t)std::max<int64_t>(n, 1));
        const RowStore::Col& sc = s.cols[c];
        if (perm && n > 0) {
            DevScope scope(p);   // the column's gather buffers
            uint8_t *tv = nullptr, *tn = nullptr; int rc;
            if ((rc = scope.alloc(&tv, (size_t)n * oc.elem))) return rc;
            if ((rc = scope.alloc(&tn, (size_t)n))) return rc;
            if ((rc = store_gather(p, sc, perm + skip, n, tv, tn))) return rc;
            CK(p, cudaMemcpyAsync(oc.values.data(), tv, (size_t)n * oc.elem, cudaMemcpyDeviceToHost, st));
            CK(p, cudaMemcpyAsync(nb.data(), tn, (size_t)n, cudaMemcpyDeviceToHost, st));
            CK(p, cudaStreamSynchronize(st));
        } else if (n > 0) {
            CK(p, cudaMemcpyAsync(oc.values.data(), sc.vals + (size_t)skip * oc.elem, (size_t)n * oc.elem, cudaMemcpyDeviceToHost, st));
            CK(p, cudaMemcpyAsync(nb.data(), sc.nulls + skip, (size_t)n, cudaMemcpyDeviceToHost, st));
            CK(p, cudaStreamSynchronize(st));
        }
        bool any = false;
        for (int64_t i = 0; i < n; i++) any |= nb[(size_t)i] != 0;
        if (any) {
            oc.validity.assign((size_t)(n + 7) / 8 + 1, 0xFF);
            for (int64_t i = 0; i < n; i++) if (nb[(size_t)i]) oc.validity[(size_t)i >> 3] &= (uint8_t)~(1u << (i & 7));
        }
        p->result.push_back(std::move(oc));
    }
    p->result_rows = n; p->result_pos = 0;
    return BKGPU_OK;
}

namespace {

// ---- exclusive prefix sum, in place, over any length (tiles of 2048, the tile sums scanned recursively) ----
constexpr int SCAN_T = 256, SCAN_I = 8, SCAN_TILE = SCAN_T * SCAN_I;

template <typename T>
__global__ void __launch_bounds__(SCAN_T) k_scan_tile(T* d, T* sums, int64_t n) {
    __shared__ T wsum[SCAN_T / 32];
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_I;
    T v[SCAN_I], acc = 0;
#pragma unroll
    for (int i = 0; i < SCAN_I; i++) { v[i] = base + i < n ? d[base + i] : T(0); acc += v[i]; }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    T x = acc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const T y = __shfl_up_sync(~0u, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[w] = x;
    __syncthreads();
    if (w == 0) {
        T s = lane < SCAN_T / 32 ? wsum[lane] : T(0);
#pragma unroll
        for (int o = 1; o < SCAN_T / 32; o <<= 1) { const T y = __shfl_up_sync(~0u, s, o); if (lane >= o) s += y; }
        if (lane < SCAN_T / 32) wsum[lane] = s;
    }
    __syncthreads();
    T run = x - acc + (w ? wsum[w - 1] : T(0));
#pragma unroll
    for (int i = 0; i < SCAN_I; i++) { if (base + i < n) d[base + i] = run; run += v[i]; }
    if (threadIdx.x == SCAN_T - 1) sums[blockIdx.x] = run;
}

template <typename T>
__global__ void k_scan_add(T* d, const T* sums, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x + SCAN_TILE; i < n; i += (int64_t)gridDim.x * blockDim.x) d[i] += sums[i / SCAN_TILE];
}

// ------------------------------------------------------------------------------------------------------------
// Stable LSD radix sort of 64-bit keys (optionally with a uint32_t id each), 8 bits per pass, one read and one write of the keys per pass
// ("Onesweep": chained scan with decoupled look-back):
//   k_rs_hist : ONE pass over the keys gives the histograms of all eight digits; a digit whose histogram has a single non-empty bin is
//               skipped (small-range keys, the NULL-rank image, descending flags, the pair keys' group and aggregate bits ...)
//   k_rs_pass : a CTA takes the next 3072-key tile (atomic ticket: tiles start in order, so the look-back never waits for a tile that has
//               not started), ranks its keys per digit (ballot-built peer masks + per-warp counters: stable), publishes the tile's digit
//               counts, looks back over the preceding tiles' published counts for its scatter bases, reorders the tile through shared
//               memory and writes digit-contiguous (coalesced) runs
// ------------------------------------------------------------------------------------------------------------
constexpr int RS_THREADS = 256;
constexpr int RS_ITEMS = 12;
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;   // 3072 keys per CTA tile (36 KB of shared memory for the reorder with ids): four CTAs per SM
constexpr uint32_t RS_FLAG_AGG = 1u << 30, RS_FLAG_PREFIX = 2u << 30, RS_VAL_MASK = (uint32_t)RADIX_MAX_KEYS;
constexpr size_t RS_HIST_BYTES = (8 * 256 * 2 + 8 + 8) * 4;   // histograms, bases, active flags, tickets

__global__ void __launch_bounds__(256) k_rs_hist(const uint64_t* key, uint32_t n, uint32_t* hist /* [8][256] */) {
    __shared__ uint32_t h[8][256];
    for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) (&h[0][0])[i] = 0;
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint64_t k = key[i];
#pragma unroll
        for (int d = 0; d < 8; d++) atomicAdd(&h[d][(k >> (8 * d)) & 0xFF], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) { const uint32_t v = (&h[0][0])[i]; if (v) atomicAdd(hist + i, v); }
}
// per digit: exclusive scan of its histogram -> global scatter bases; active[d] = more than one non-empty bin
__global__ void k_rs_bases(const uint32_t* hist, uint32_t* bases, uint32_t* active) {
    const int d = blockIdx.x;
    __shared__ uint32_t s[256];
    const uint32_t v = hist[d * 256 + threadIdx.x];
    s[threadIdx.x] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t run = 0, nz = 0;
        for (int i = 0; i < 256; i++) { const uint32_t c = s[i]; s[i] = run; run += c; nz += c != 0; }
        active[d] = nz > 1;
    }
    __syncthreads();
    bases[d * 256 + threadIdx.x] = s[threadIdx.x];
}

// IDS == false: id_in / id_out are not touched, and the tile's ids take no shared memory
template <bool IDS>
__global__ void __launch_bounds__(RS_THREADS, 4) k_rs_pass(const uint64_t* key_in, const uint32_t* id_in, uint64_t* key_out, uint32_t* id_out, uint32_t n, int shift,
                                                        const uint32_t* global_base /* [256] of this digit */, uint32_t* status /* [ntiles][256], zeroed */,
                                                        uint32_t* ticket) {
    extern __shared__ __align__(16) unsigned char rs_smem[];
    uint64_t* s_key = (uint64_t*)rs_smem;                        // [RS_TILE]
    uint32_t* s_id = (uint32_t*)(s_key + RS_TILE);               // [RS_TILE] (IDS)
    uint32_t* wcnt = s_id + (IDS ? RS_TILE : 0);                 // [8][256] per-warp digit counts -> running offsets inside the digit's run
    uint32_t* dstart = wcnt + 8 * 256;                           // [256] start of the digit inside the reordered tile
    uint32_t* tbase = dstart + 256;                              // [256] global address of the tile's first key of the digit
    __shared__ uint32_t s_tile;
    __shared__ uint32_t wsum[8];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
    for (int i = threadIdx.x; i < 8 * 256; i += RS_THREADS) wcnt[i] = 0;
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint32_t t0 = tile * RS_TILE;
    const uint32_t tile_n = min((uint32_t)RS_TILE, n - t0);
    // ---- load: warp w owns the contiguous chunk [t0 + w * 32 * RS_ITEMS, + 32 * RS_ITEMS), RS_ITEMS rounds of 32 consecutive keys ----
    uint64_t k[RS_ITEMS]; uint32_t id[RS_ITEMS];
    const uint32_t c0 = w * (RS_ITEMS * 32);
#pragma unroll
    for (int r = 0; r < RS_ITEMS; r++) {
        const uint32_t li = c0 + r * 32 + lane;
        if (li < tile_n) { k[r] = key_in[t0 + li]; if (IDS) id[r] = id_in[t0 + li]; } else { k[r] = ~0ull; id[r] = 0; }
    }
    // ---- early counts: the warp's digit histogram (order-free atomics), so the tile's counts are published BEFORE the ranking and the
    //      following tiles' look-back finds them sooner ----
    uint32_t* wc = wcnt + w * 256;
#pragma unroll
    for (int r = 0; r < RS_ITEMS; r++)
        if (c0 + r * 32 + lane < tile_n) atomicAdd(wc + (uint32_t)((k[r] >> shift) & 0xFF), 1u);
    __syncthreads();
    // ---- thread d: the digit's count per warp -> per-warp offsets, tile count; publish; where the digit starts in the reordered tile ----
    const int d_own = threadIdx.x;
    uint32_t cnt;
    volatile uint32_t* st = status + (size_t)tile * 256 + d_own;
    {
        uint32_t run = 0;
#pragma unroll
        for (int ww = 0; ww < 8; ww++) { const uint32_t c = wcnt[ww * 256 + d_own]; wcnt[ww * 256 + d_own] = run; run += c; }
        cnt = run;
        *st = (tile == 0 ? RS_FLAG_PREFIX : RS_FLAG_AGG) | cnt;   // (flag and count travel in ONE word: no fence around the publication)
        uint32_t x = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o); if (lane >= o) x += y; }
        if (lane == 31) wsum[w] = x;
        __syncthreads();
        uint32_t wpre = 0;
        for (int ww = 0; ww < w; ww++) wpre += wsum[ww];
        dstart[d_own] = wpre + x - cnt;
    }
    __syncthreads();
    // ---- rank in element order (stable) and place: peers of the digit in this round + the digit's running offset.  The peer mask
    //      comes from eight ballots, one per digit bit: MATCH.ANY would keep the XU pipe busy ----
    const uint32_t lt_mask = (1u << lane) - 1u;
#pragma unroll
    for (int r = 0; r < RS_ITEMS; r++) {
        const bool live = c0 + r * 32 + lane < tile_n;
        const uint32_t d = (uint32_t)((k[r] >> shift) & 0xFF);
        uint32_t peers = __ballot_sync(0xFFFFFFFFu, live);
#pragma unroll
        for (int b = 0; b < 8; b++) {
            const uint32_t bit = (d >> b) & 1u;
            peers &= ~(__ballot_sync(0xFFFFFFFFu, bit != 0) ^ (0u - bit));
        }
        uint32_t before = 0;
        if (live) before = wc[d];
        __syncwarp();
        const uint32_t mine = __popc(peers & lt_mask);
        if (live) {
            if ((peers >> lane) == 1u) wc[d] = before + mine + 1u;   // the highest peer lane advances the offset by the group's size
            const uint32_t pos = dstart[d] + before + mine;
            s_key[pos] = k[r]; if (IDS) s_id[pos] = id[r];
        }
        __syncwarp();
    }
    // ---- chained scan with decoupled look-back over the preceding tiles (they all started before this one: ticket order) ----
    {
        uint32_t excl = 0;
        if (tile != 0) {
            // four predecessors per round trip: the loads are independent, the walk consumes them nearest first
            for (int64_t p = (int64_t)tile - 1;;) {
                uint32_t v[4];
#pragma unroll
                for (int j = 0; j < 4; j++) v[j] = p - j >= 0 ? *(volatile const uint32_t*)(status + (size_t)(p - j) * 256 + d_own) : RS_FLAG_PREFIX;
                int j = 0; bool done = false;
#pragma unroll
                for (; j < 4; j++) {
                    if ((v[j] & ~RS_VAL_MASK) == 0) break;            // not published yet: poll again from this tile
                    excl += v[j] & RS_VAL_MASK;
                    if (v[j] & RS_FLAG_PREFIX) { done = true; break; }
                }
                if (done) break;
                p -= j;
            }
            *st = RS_FLAG_PREFIX | (excl + cnt);
        }
        tbase[d_own] = global_base[d_own] + excl;
    }
    __syncthreads();
    // ---- write the digit-contiguous runs ----
    for (uint32_t i = threadIdx.x; i < tile_n; i += RS_THREADS) {
        const uint64_t kk = s_key[i];
        const uint32_t d = (uint32_t)((kk >> shift) & 0xFF);
        const uint32_t dst = tbase[d] + (i - dstart[d]);
        key_out[dst] = kk; if (IDS) id_out[dst] = s_id[i];
    }
}

}  // namespace

int64_t scan_scratch(int64_t n) { int64_t t = 0; while (n > 1) { n = (n + SCAN_TILE - 1) / SCAN_TILE; t += n; } return t + 1; }

template <typename T>
cudaError_t scan_excl(T* d, int64_t n, T* sums, int sm, cudaStream_t s) {
    const int64_t nb = (n + SCAN_TILE - 1) / SCAN_TILE;
    k_scan_tile<T><<<(unsigned)nb, SCAN_T, 0, s>>>(d, sums, n);
    if (nb > 1) {
        cudaError_t e = scan_excl(sums, nb, sums + nb, sm, s);
        if (e != cudaSuccess) return e;
        k_scan_add<T><<<grid_for(n, sm, 16), 256, 0, s>>>(d, sums, n);
    }
    return cudaGetLastError();
}
template cudaError_t scan_excl<uint32_t>(uint32_t*, int64_t, uint32_t*, int, cudaStream_t);
template cudaError_t scan_excl<uint64_t>(uint64_t*, int64_t, uint64_t*, int, cudaStream_t);

int radix_sort(bkgpu_plan* p, uint64_t* const keys[2], uint32_t* const ids[2], int cur, int64_t n, RadixScratch& scratch, bkgpu_stats* stats,
               int64_t* bytes) {
    if (n > RADIX_MAX_KEYS) return p->fail(BKGPU_EUNSUPPORTED, "the radix sort takes at most 2^30 - 1 keys");
    if (n < 2) return cur;
    const cudaStream_t st = p->stream;
    const int sm = p->sm_count;
    const uint32_t un = (uint32_t)n, ntiles = (un + RS_TILE - 1) / RS_TILE;
    int rc;
    if ((rc = ensure_buf(p, &scratch.hist, &scratch.hist_cap, RS_HIST_BYTES))) return rc;
    uint32_t* hist = (uint32_t*)scratch.hist;
    uint32_t* bases = hist + 8 * 256; uint32_t* active = bases + 8 * 256; uint32_t* tickets = active + 8;
    CK(p, cudaMemsetAsync(hist, 0, RS_HIST_BYTES, st));
    k_rs_hist<<<std::min(sm * 4, (int)((un + 1023) / 1024)), 256, 0, st>>>(keys[cur], un, hist);
    k_rs_bases<<<8, 256, 0, st>>>(hist, bases, active);
    uint32_t h_active[8];
    CK(p, cudaMemcpyAsync(h_active, active, 32, cudaMemcpyDeviceToHost, st));
    CK(p, cudaStreamSynchronize(st));
    stats->kernel_launches += 2;
    if (bytes) *bytes += n * 8;
    int n_active = 0;
    for (int d = 0; d < 8; d++) n_active += h_active[d] != 0;
    if (!n_active) return cur;
    const size_t status_bytes = (size_t)ntiles * 256 * 4 * (size_t)n_active;   // one look-back array per pass
    if ((rc = ensure_buf(p, &scratch.status, &scratch.status_cap, status_bytes))) return rc;
    uint32_t* status = (uint32_t*)scratch.status;
    CK(p, cudaMemsetAsync(status, 0, status_bytes, st));
    const auto pass = ids ? k_rs_pass<true> : k_rs_pass<false>;
    const size_t smem = (size_t)RS_TILE * (ids ? 12 : 8) + (8 * 256 + 256 + 256) * 4;   // under 48 KB: no opt-in needed
    int slot = 0;
    for (int d = 0; d < 8; d++) {
        if (!h_active[d]) continue;
        pass<<<ntiles, RS_THREADS, smem, st>>>(keys[cur], ids ? ids[cur] : nullptr, keys[cur ^ 1], ids ? ids[cur ^ 1] : nullptr, un, 8 * d,
                                               bases + 256 * d, status + (size_t)slot * ntiles * 256, tickets + d);
        cur ^= 1; slot++;
        stats->kernel_launches++;
        if (bytes) *bytes += n * (ids ? 24 : 16);
    }
    CK(p, cudaGetLastError());
    return cur;
}

}  // namespace bk

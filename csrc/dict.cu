// dict.cu — the order-preserving dictionary of STRING columns, built on the device (bkgpu_dict_*, include/bkgpu.h), for sm_90a.
//
// One comparison domain — one or more large_binary columns in device memory — becomes its sorted distinct values and one INT32 code column
// per input column, the code of a value being its rank in that sorted list (a NULL: code 0, validity bit clear).  Order: unsigned bytes,
// a proper prefix first (std::string::compare, Arrow's sort of binary values).
//   1. deduplicate: every non-NULL string is hashed into an open-addressing table of (64-bit hash, representative row); a thread hashes a
//      string of at most LONG_BYTES bytes, a warp a longer one.  Equal hashes are confirmed byte by byte before two rows share a value.
//   2. sort the distinct values by MSD rounds over 8-byte big-endian chunks: round k sorts only the values whose segment (the values tied
//      on the first 8k bytes) still has more than one member, by (segment, chunk k, min(len - 8k, 9)), with the library's stable radix
//      sort (prims.cu): once by the key's low word, then by its high word.  The last field puts "ab" before "ab\0" and ends a value's
//      refinement; the rounds stop when no segment has two members, after (longest shared prefix) / 8 + 1 rounds.
//   3. rank = position after the sort; code[row] = rank of the row's value.
// The handle owns a bkgpu_plan without a compiled fragment for its stream, its allocator and its error reporting.
#include <string.h>
#include <algorithm>
#include <vector>
#include "api_state.h"
#include "prims.cuh"

namespace {

constexpr uint64_t EMPTY_KEY = ~0ull;
constexpr uint32_t NONE = 0xFFFFFFFFu;      // empty table slot / NULL row
constexpr int64_t LONG_BYTES = 64;          // longer strings are hashed and compared by a warp
constexpr int64_t MAX_ROWS = (int64_t)1 << 30;

// the 8 bytes of s at `at` as a big-endian word, zero past the end: unsigned comparison of two words = byte-wise comparison
__device__ __forceinline__ uint64_t chunk_be(const uint8_t* s, int64_t len, int64_t at) {
    uint64_t v = 0;
    if (at + 8 <= len) {
#pragma unroll
        for (int b = 0; b < 8; b++) v = v << 8 | s[at + b];
    } else {
        for (int b = 0; b < 8; b++) v = v << 8 | (at + b < len ? s[at + b] : 0u);
    }
    return v;
}

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}
// chunk i's share of the hash: a sum of independent terms, so a warp reduces the terms its lanes hashed in any order
__device__ __forceinline__ uint64_t chunk_term(uint64_t c, int64_t i) { return mix64(c + (uint64_t)i * 0x9E3779B97F4A7C15ull); }
__device__ __forceinline__ uint64_t finish_hash(uint64_t acc, int64_t len, uint64_t hmask) {
    uint64_t h = mix64(acc ^ ((uint64_t)len * 0xD6E8FEB86659FD93ull)) & hmask;
    return h == EMPTY_KEY ? EMPTY_KEY - 1 : h;
}

// one column of the domain -> per row (global row base + i): the string's address and length, -1 for a NULL
__global__ void k_resolve(const int64_t* off, const uint8_t* data, const uint8_t* valid, int64_t voff, int64_t n, uint64_t* sptr, int64_t* slen) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = voff + i;
        const bool ok = !valid || ((valid[b >> 3] >> (b & 7)) & 1);
        const int64_t o0 = off[i];
        sptr[i] = (uint64_t)(uintptr_t)(data + o0);
        slen[i] = ok ? off[i + 1] - o0 : -1;
    }
}

// The table: keys[s] a hash (EMPTY_KEY: free), rows[s] the row that claimed it (NONE until its claimer has written it).  Two rows share a
// value only when their bytes are equal; an equal hash with different bytes probes on.
__device__ __forceinline__ uint32_t claimed_row(const uint32_t* rows, uint64_t s) {
    uint32_t r;
    while ((r = *(volatile const uint32_t*)(rows + s)) == NONE) {}
    return r;
}

__global__ void __launch_bounds__(256) k_dedup(const uint64_t* sptr, const int64_t* slen, int64_t n, uint64_t* keys, uint32_t* rows, uint64_t mask,
                                               uint64_t hmask, uint32_t* sid) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + threadIdx.x - lane; base < n; base += stride) {
        const int64_t r = base + lane;
        const int64_t len = r < n ? slen[r] : -1;
        // ---- a short string: this thread ----
        if (r < n && len < 0) sid[r] = NONE;
        if (r < n && len >= 0 && len <= LONG_BYTES) {
            const uint8_t* s = (const uint8_t*)(uintptr_t)sptr[r];
            uint64_t acc = 0;
            for (int64_t i = 0; i * 8 < len; i++) acc += chunk_term(chunk_be(s, len, i * 8), i);
            const uint64_t h = finish_hash(acc, len, hmask);
            for (uint64_t at = h & mask;; at = (at + 1) & mask) {
                uint64_t k = keys[at];
                if (k == EMPTY_KEY) {
                    k = atomicCAS((unsigned long long*)(keys + at), (unsigned long long)EMPTY_KEY, (unsigned long long)h);
                    if (k == EMPTY_KEY) { *(volatile uint32_t*)(rows + at) = (uint32_t)r; sid[r] = (uint32_t)at; break; }
                }
                if (k != h) continue;
                const uint32_t o = claimed_row(rows, at);
                if (slen[o] != len) continue;
                const uint8_t* t = (const uint8_t*)(uintptr_t)sptr[o];
                int64_t i = 0;
                while (i < len && s[i] == t[i]) i++;
                if (i == len) { sid[r] = (uint32_t)at; break; }
            }
        }
        // ---- the warp's long strings, one at a time, by the whole warp ----
        uint32_t todo = __ballot_sync(~0u, len > LONG_BYTES);
        while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const int64_t rr = base + src;
            const int64_t ln = __shfl_sync(~0u, len, src);
            const uint8_t* s = (const uint8_t*)(uintptr_t)sptr[rr];
            uint64_t acc = 0;
            for (int64_t i = lane; i * 8 < ln; i += 32) acc += chunk_term(chunk_be(s, ln, i * 8), i);
#pragma unroll
            for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(~0u, acc, o);
            const uint64_t h = finish_hash(acc, ln, hmask);
            for (uint64_t at = h & mask;; at = (at + 1) & mask) {
                uint32_t o = NONE;   // the row to compare with; rr itself when this warp claimed the slot, NONE for another hash
                if (lane == 0) {
                    uint64_t k = keys[at];
                    if (k == EMPTY_KEY) k = atomicCAS((unsigned long long*)(keys + at), (unsigned long long)EMPTY_KEY, (unsigned long long)h);
                    if (k == EMPTY_KEY) { *(volatile uint32_t*)(rows + at) = (uint32_t)rr; o = (uint32_t)rr; }
                    else if (k == h) o = claimed_row(rows, at);
                }
                o = __shfl_sync(~0u, o, 0);
                if (o == (uint32_t)rr) { if (lane == 0) sid[rr] = (uint32_t)at; break; }
                if (o == NONE || slen[o] != ln) continue;
                const uint8_t* t = (const uint8_t*)(uintptr_t)sptr[o];
                bool diff = false;
                for (int64_t i = lane; i < ln && !diff; i += 32) diff = s[i] != t[i];
                if (!__any_sync(~0u, diff)) { if (lane == 0) sid[rr] = (uint32_t)at; break; }
            }
        }
    }
}

// the claimed slots -> the distinct values: their representative row and slot (in any order: the sort decides)
__global__ void k_compact(const uint32_t* rows, uint64_t cap, uint32_t* rep_row, uint32_t* rep_slot, uint32_t* count) {
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = rows[s];
        if (r == NONE) continue;
        const uint32_t k = atomicAdd(count, 1u);
        rep_row[k] = r; rep_slot[k] = (uint32_t)s;
    }
}

// ---- the sort's rounds.  seg[pos]: the position where the segment of the value at sorted position pos starts ----
__device__ __forceinline__ bool tied(const uint32_t* seg, int64_t i, int64_t d) {
    return (i > 0 && seg[i - 1] == seg[i]) || (i + 1 < d && seg[i + 1] == seg[i]);
}
__global__ void k_tied_flags(const uint32_t* seg, int64_t d, uint32_t* flag) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= d; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = i < d && tied(seg, i, d) ? 1u : 0u;
}
__global__ void k_tied_list(const uint32_t* seg, int64_t d, const uint32_t* at, uint32_t* act) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < d; i += (int64_t)gridDim.x * blockDim.x)
        if (tied(seg, i, d)) act[at[i]] = (uint32_t)i;
}
// key of active value j at byte depth `depth`: high word (segment, chunk bytes 0..3), low word (chunk bytes 4..7, min(len - depth, 9))
__global__ void k_round_keys(const uint32_t* act, int64_t a, const uint32_t* order, const uint32_t* seg, const uint32_t* rep_row, const uint64_t* sptr,
                             const int64_t* slen, int64_t depth, uint64_t* kh, uint64_t* kl, uint64_t* kl_sort, uint32_t* ids) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a; j += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t pos = act[j];
        const uint32_t r = rep_row[order[pos]];
        const int64_t len = slen[r];
        const uint64_t c = chunk_be((const uint8_t*)(uintptr_t)sptr[r], len, depth);
        const uint64_t tail = (uint64_t)std::min<int64_t>(std::max<int64_t>(len - depth, 0), 9);
        kh[j] = (uint64_t)seg[pos] << 32 | c >> 32;
        kl[j] = kl_sort[j] = (c & 0xFFFFFFFFull) << 4 | tail;
        ids[j] = (uint32_t)j;
    }
}
__global__ void k_gather_u64(const uint64_t* src, const uint32_t* ids, int64_t n, uint64_t* dst) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) dst[t] = src[ids[t]];
}
__device__ __forceinline__ bool group_head(const uint32_t* perm, const uint64_t* kh, const uint64_t* kl, int64_t t) {
    return t == 0 || kh[perm[t]] != kh[perm[t - 1]] || kl[perm[t]] != kl[perm[t - 1]];
}
// after the round's sort (perm): the value that lands on active slot t, and whether t starts a new group
__global__ void k_round_heads(const uint32_t* perm, const uint64_t* kh, const uint64_t* kl, int64_t a, const uint32_t* act, const uint32_t* order,
                              uint32_t* moved, uint32_t* head) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t <= a; t += (int64_t)gridDim.x * blockDim.x) {
        if (t == a) { head[t] = 0; continue; }
        moved[t] = order[act[perm[t]]];
        head[t] = group_head(perm, kh, kl, t) ? 1u : 0u;
    }
}
__global__ void k_group_starts(const uint32_t* perm, const uint64_t* kh, const uint64_t* kl, int64_t a, const uint32_t* ord, uint32_t* gstart) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < a; t += (int64_t)gridDim.x * blockDim.x)
        if (group_head(perm, kh, kl, t)) gstart[ord[t]] = (uint32_t)t;
}
// the active slots are the whole positions of their segments, in position order, and the sort keeps segments apart: active slot t is
// position act[t]
__global__ void k_round_scatter(const uint32_t* perm, const uint64_t* kh, const uint64_t* kl, int64_t a, const uint32_t* act, const uint32_t* moved,
                                const uint32_t* ord, const uint32_t* gstart, uint32_t* order, uint32_t* seg) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < a; t += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t g = ord[t] + (group_head(perm, kh, kl, t) ? 1u : 0u) - 1u;
        order[act[t]] = moved[t];
        seg[act[t]] = act[gstart[g]];
    }
}

// ---- rank, codes and the dictionary ----
__global__ void k_slot_rank(const uint32_t* order, const uint32_t* rep_slot, int64_t d, uint32_t* slot_rank) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < d; i += (int64_t)gridDim.x * blockDim.x) slot_rank[rep_slot[order[i]]] = (uint32_t)i;
}
__global__ void k_row_codes(uint32_t* sid, int64_t n, const uint32_t* slot_rank) {   // in place: slot -> rank (NONE stays: a NULL)
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t s = sid[i];
        if (s != NONE) sid[i] = slot_rank[s];
    }
}
__global__ void k_dict_lengths(const uint32_t* order, const uint32_t* rep_row, const int64_t* slen, int64_t d, uint64_t* off) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= d; i += (int64_t)gridDim.x * blockDim.x)
        off[i] = i < d ? (uint64_t)slen[rep_row[order[i]]] : 0;
}
__global__ void k_dict_bytes(const uint32_t* order, const uint32_t* rep_row, const uint64_t* sptr, int64_t d, const uint64_t* off, uint8_t* out) {
    const int lane = threadIdx.x & 31;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < d; i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        const uint8_t* s = (const uint8_t*)(uintptr_t)sptr[rep_row[order[i]]];
        const uint64_t o = off[i], len = off[i + 1] - o;
        for (uint64_t b = lane; b < len; b += 32) out[o + b] = s[b];
    }
}
// one column's codes (NULL -> 0) and its validity bitmap from bit 0; *nulls counts the NULLs
__global__ void k_column_codes(const uint32_t* code, int64_t n, int32_t* out, uint8_t* validity, unsigned long long* nulls) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < (n + 7) / 8; b += (int64_t)gridDim.x * blockDim.x) {
        uint32_t v = 0, nn = 0;
        for (int j = 0; j < 8 && b * 8 + j < n; j++) {
            const uint32_t c = code[b * 8 + j];
            out[b * 8 + j] = c == NONE ? 0 : (int32_t)c;
            if (c == NONE) nn++; else v |= 1u << j;
        }
        if (validity) validity[b] = (uint8_t)v;
        if (nn) atomicAdd(nulls, (unsigned long long)nn);
    }
}

int fail_thread(int code, const char* msg) { g_thread_error = msg; return code; }

}  // namespace

struct bkgpu_dict {
    bkgpu_plan* p = nullptr;               // stream, allocator, error reporting (no compiled fragment)
    std::vector<int64_t> base, len;        // each column's first row in `codes`, and its rows
    uint32_t* codes = nullptr;             // per row of the domain: the rank, NONE for a NULL
    uint64_t* dict_off = nullptr;          // n_values + 1 offsets from 0
    uint8_t* dict_bytes = nullptr;
    int64_t n_values = 0, n_bytes = 0;
};

namespace {

int dict_build(bkgpu_dict* d, const bkgpu_binary_column* cols, int ncols, int hash_bits) {
    bkgpu_plan* p = d->p;
    const cudaStream_t st = p->stream;
    const int sm = p->sm_count;
    int64_t n = 0;
    for (int c = 0; c < ncols; c++) { d->base.push_back(n); d->len.push_back(cols[c].length); n += cols[c].length; }
    if (n > MAX_ROWS) return p->fail(BKGPU_EUNSUPPORTED, "a dictionary domain of more than 2^30 rows is outside the GPU path");
    int rc;
    if ((rc = dev_alloc(p, (void**)&d->codes, (size_t)std::max<int64_t>(n, 1) * 4))) return rc;
    DevScope scope(p);   // everything else is the build's
    uint64_t* sptr; int64_t* slen;
    if ((rc = scope.alloc(&sptr, (size_t)std::max<int64_t>(n, 1) * 8)) || (rc = scope.alloc(&slen, (size_t)std::max<int64_t>(n, 1) * 8))) return rc;
    for (int c = 0; c < ncols; c++)
        if (cols[c].length > 0)
            k_resolve<<<grid_for(cols[c].length, sm, 8), 256, 0, st>>>(cols[c].offsets, cols[c].data, cols[c].validity, cols[c].validity_offset,
                                                                        cols[c].length, sptr + d->base[c], slen + d->base[c]);
    // ---- 1. deduplicate ----
    uint64_t cap = 1024;
    while (cap < (uint64_t)n * 2) cap <<= 1;
    uint64_t* keys; uint32_t* rows; uint32_t* counter;
    if ((rc = scope.alloc(&keys, cap * 8)) || (rc = scope.alloc(&rows, cap * 4)) || (rc = scope.alloc(&counter, 64))) return rc;
    CK(p, cudaMemsetAsync(keys, 0xFF, cap * 8, st));
    CK(p, cudaMemsetAsync(rows, 0xFF, cap * 4, st));
    CK(p, cudaMemsetAsync(counter, 0, 64, st));
    const uint64_t hmask = hash_bits >= 64 || hash_bits <= 0 ? ~0ull : ((1ull << hash_bits) - 1);
    if (n > 0) k_dedup<<<grid_for(n, sm, 8), 256, 0, st>>>(sptr, slen, n, keys, rows, cap - 1, hmask, d->codes);
    uint32_t* rep_row; uint32_t* rep_slot;
    if ((rc = scope.alloc(&rep_row, (size_t)std::max<int64_t>(n, 1) * 4)) || (rc = scope.alloc(&rep_slot, (size_t)std::max<int64_t>(n, 1) * 4))) return rc;
    k_compact<<<grid_for((int64_t)cap, sm, 8), 256, 0, st>>>(rows, cap, rep_row, rep_slot, counter);
    CK(p, cudaGetLastError());
    uint32_t dcount = 0;
    CK(p, cudaMemcpyAsync(&dcount, counter, 4, cudaMemcpyDeviceToHost, st));
    CK(p, cudaStreamSynchronize(st));
    const int64_t dn = dcount;
    if (dn >= (int64_t)1 << 31) return p->fail(BKGPU_EUNSUPPORTED, "more than 2^31 distinct strings in one comparison domain");
    // ---- 2. sort the distinct values ----
    const size_t dsz = (size_t)std::max<int64_t>(dn, 1) + 1;
    uint32_t *order, *seg, *flag, *act, *moved, *ids[2], *gstart;
    uint64_t *kh, *kl, *ksort[2];
    if ((rc = scope.alloc(&order, dsz * 4)) || (rc = scope.alloc(&seg, dsz * 4)) || (rc = scope.alloc(&flag, dsz * 4)) || (rc = scope.alloc(&act, dsz * 4)) ||
        (rc = scope.alloc(&moved, dsz * 4)) || (rc = scope.alloc(&ids[0], dsz * 4)) || (rc = scope.alloc(&ids[1], dsz * 4)) || (rc = scope.alloc(&gstart, dsz * 4)) ||
        (rc = scope.alloc(&kh, dsz * 8)) || (rc = scope.alloc(&kl, dsz * 8)) || (rc = scope.alloc(&ksort[0], dsz * 8)) || (rc = scope.alloc(&ksort[1], dsz * 8)))
        return rc;
    uint32_t* sums;
    if ((rc = scope.alloc(&sums, (size_t)scan_scratch((int64_t)dsz) * 4))) return rc;
    if (dn > 0) k_iota<<<grid_for(dn, sm, 8), 256, 0, st>>>(order, dn);
    CK(p, cudaMemsetAsync(seg, 0, dsz * 4, st));
    RadixScratch rs;   // (the plan's buffers: bkgpu_dict_free returns them on a failure)
    for (int64_t depth = 0; dn > 1; depth += 8) {
        k_tied_flags<<<grid_for(dn + 1, sm, 8), 256, 0, st>>>(seg, dn, flag);
        CK(p, scan_excl<uint32_t>(flag, dn + 1, sums, sm, st));
        k_tied_list<<<grid_for(dn, sm, 8), 256, 0, st>>>(seg, dn, flag, act);
        uint32_t na = 0;
        CK(p, cudaMemcpyAsync(&na, flag + dn, 4, cudaMemcpyDeviceToHost, st));
        CK(p, cudaStreamSynchronize(st));
        p->stats.kernel_launches += 2;
        if (!na) break;
        const int64_t a = na;
        k_round_keys<<<grid_for(a, sm, 8), 256, 0, st>>>(act, a, order, seg, rep_row, sptr, slen, depth, kh, kl, ksort[0], ids[0]);
        // (segment, chunk, tail): stable by the low word, then by the high word
        uint64_t* const kb[2] = {ksort[0], ksort[1]};
        const int c1 = radix_sort(p, kb, ids, 0, a, rs, &p->stats, nullptr);
        if (c1 < 0) return c1;
        k_gather_u64<<<grid_for(a, sm, 8), 256, 0, st>>>(kh, ids[c1], a, ksort[c1]);
        const int c2 = radix_sort(p, kb, ids, c1, a, rs, &p->stats, nullptr);
        if (c2 < 0) return c2;
        const uint32_t* perm = ids[c2];
        k_round_heads<<<grid_for(a + 1, sm, 8), 256, 0, st>>>(perm, kh, kl, a, act, order, moved, flag);
        CK(p, scan_excl<uint32_t>(flag, a + 1, sums, sm, st));
        k_group_starts<<<grid_for(a, sm, 8), 256, 0, st>>>(perm, kh, kl, a, flag, gstart);
        k_round_scatter<<<grid_for(a, sm, 8), 256, 0, st>>>(perm, kh, kl, a, act, moved, flag, gstart, order, seg);
        CK(p, cudaGetLastError());
        p->stats.kernel_launches += 6;
    }
    dev_free(p, rs.hist); dev_free(p, rs.status);
    // ---- 3. rank, codes, the dictionary ----
    uint32_t* slot_rank = rows;   // (the table's rows are no longer read)
    if (dn > 0) k_slot_rank<<<grid_for(dn, sm, 8), 256, 0, st>>>(order, rep_slot, dn, slot_rank);
    if (n > 0) k_row_codes<<<grid_for(n, sm, 8), 256, 0, st>>>(d->codes, n, slot_rank);
    if ((rc = dev_alloc(p, (void**)&d->dict_off, (size_t)(dn + 1) * 8))) return rc;
    uint64_t* sums64;
    if ((rc = scope.alloc(&sums64, (size_t)scan_scratch(dn + 1) * 8))) return rc;
    k_dict_lengths<<<grid_for(dn + 1, sm, 8), 256, 0, st>>>(order, rep_row, slen, dn, d->dict_off);
    CK(p, scan_excl<uint64_t>(d->dict_off, dn + 1, sums64, sm, st));
    uint64_t total = 0;
    CK(p, cudaMemcpyAsync(&total, d->dict_off + dn, 8, cudaMemcpyDeviceToHost, st));
    CK(p, cudaStreamSynchronize(st));
    if ((rc = dev_alloc(p, (void**)&d->dict_bytes, (size_t)std::max<uint64_t>(total, 1)))) return rc;
    if (dn > 0) k_dict_bytes<<<grid_for(dn * 32, sm, 8), 256, 0, st>>>(order, rep_row, sptr, dn, d->dict_off, d->dict_bytes);
    CK(p, cudaGetLastError());
    CK(p, cudaStreamSynchronize(st));
    p->stats.kernel_launches += 8;
    d->n_values = dn; d->n_bytes = (int64_t)total;
    return BKGPU_OK;
}

}  // namespace

extern "C" int bkgpu_dict_build(bkgpu_dict** out, int device, void* stream, const bkgpu_binary_column* cols, int ncols, int hash_bits) {
    if (!out) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_build: out is NULL");
    *out = nullptr;
    if (!cols || ncols < 1) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_build: no columns");
    if (hash_bits < 0 || hash_bits > 64) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_build: hash_bits out of range (0 .. 64)");
    for (int c = 0; c < ncols; c++) {
        if (cols[c].length < 0) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_build: negative column length");
        if (cols[c].validity_offset < 0) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_build: negative validity offset");
        if (!cols[c].offsets || !cols[c].data) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_build: NULL offsets or data");
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) {
        g_thread_error = std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") + " (this library has no CPU fallback)";
        return BKGPU_ENODEV;
    }
    if (device < 0 || device >= ndev) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_build: bad device index");
    bkgpu_dict* d = new bkgpu_dict();
    d->p = new bkgpu_plan();
    bkgpu_plan* p = d->p;
    p->device = device;
    { int n = 0; if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && n > 0) p->sm_count = n; }
    int rc = BKGPU_OK;
    if ((e = cudaSetDevice(device)) != cudaSuccess) rc = p->cuda_fail(e, "cudaSetDevice");
    else if (stream) p->stream = (cudaStream_t)stream;
    else if ((e = cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking)) != cudaSuccess) rc = p->cuda_fail(e, "cudaStreamCreateWithFlags");
    else p->own_stream = true;
    if (!rc) rc = dict_build(d, cols, ncols, hash_bits);
    if (rc) { bkgpu_dict_free(d); return rc; }   // (the message stays in the thread's error: bkgpu_last_error(NULL))
    p->state = S_FINISHED;
    *out = d;
    return BKGPU_OK;
}

extern "C" int bkgpu_dict_size(bkgpu_dict* d, int64_t* n_values, int64_t* n_bytes) {
    if (!d || !n_values || !n_bytes) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_size: NULL argument");
    *n_values = d->n_values; *n_bytes = d->n_bytes;
    return BKGPU_OK;
}

extern "C" int bkgpu_dict_copy(bkgpu_dict* d, int64_t* offsets, uint8_t* bytes, int on_device) {
    if (!d || !offsets || (!bytes && d->n_bytes > 0)) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_copy: NULL argument");
    bkgpu_plan* p = d->p;
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    CK(p, cudaSetDevice(p->device));
    CK(p, cudaMemcpyAsync(offsets, d->dict_off, (size_t)(d->n_values + 1) * 8, kind, p->stream));
    if (d->n_bytes > 0) CK(p, cudaMemcpyAsync(bytes, d->dict_bytes, (size_t)d->n_bytes, kind, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    return BKGPU_OK;
}

extern "C" int bkgpu_dict_codes(bkgpu_dict* d, int column, int32_t* codes, uint8_t* validity, int64_t* null_count) {
    if (!d) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_codes: NULL handle");
    if (column < 0 || column >= (int)d->len.size()) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_codes: no such column");
    bkgpu_plan* p = d->p;
    const int64_t n = d->len[column];
    if (!codes && n > 0) return fail_thread(BKGPU_EINVAL, "bkgpu_dict_codes: NULL codes");
    CK(p, cudaSetDevice(p->device));
    unsigned long long* cnt;
    DevScope scope(p);
    int rc;
    if ((rc = scope.alloc(&cnt, 8))) return rc;
    CK(p, cudaMemsetAsync(cnt, 0, 8, p->stream));
    if (n > 0) k_column_codes<<<grid_for((n + 7) / 8, p->sm_count, 8), 256, 0, p->stream>>>(d->codes + d->base[column], n, codes, validity, cnt);
    CK(p, cudaGetLastError());
    unsigned long long nn = 0;
    CK(p, cudaMemcpyAsync(&nn, cnt, 8, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    if (null_count) *null_count = (int64_t)nn;
    return BKGPU_OK;
}

extern "C" void bkgpu_dict_free(bkgpu_dict* d) {
    if (!d) return;
    if (d->p) bkgpu_close(d->p);   // drains the stream, returns every buffer to the allocator's cache, destroys a stream it created
    delete d;
}

// join.cu — the hash join (K4): its kernels (multimap and unique-key index builds, gathers, the star join's filter, probe and expansion) and
// its host path: the retained build sides and their indexes, the two-table probe (fused into the lean aggregate, gather, general), the
// outer-join tail, the join that returns rows, and the star join's build and probe.  The probe loops that run the row interpreter over the
// joined row (k_agg_interp, k_join_pairs) are agg.cu's.
#include <string.h>
#include <algorithm>
#include <vector>
#include "api_state.h"
#include "dev_common.cuh"
#include "interp.cuh"

namespace bk {

// build-side columns gathered to probe-row alignment (k_join_gather): elements of 8, 4, 16 (a STRING slot: the AVG blob a MERGE_AGG over
// the join reads) or 1 byte
struct GatherCols { int32_t n; const uint8_t* src[MAX_COLS]; uint8_t* dst[MAX_COLS]; int32_t elem[MAX_COLS]; };
// star join (PK_STAR_AGG): per dimension with unique keys, the fact foreign key, its slot in the row-id tuple and the dimension's key index
struct StarLookup { DevCol fk; int32_t from_prim, cast_prim, slot; JoinFast jf; };
struct StarProbe { StarLookup d[4]; int32_t n; int32_t width; int64_t nrows; int32_t vec; };
// the build-time filter of one dimension: program over the plan's columns (this dimension's retained rows), validity of its join key.
// Also a two-table join child's own filter (its retained build rows, or one probe batch).
struct StarFilter { DevCol cols[MAX_COLS]; Program prog; int32_t key_col; int64_t nrows; };

// one output column of the joined rows: element `which` of each row-id tuple (`width` row ids: (probe, build) pairs of a two-table join,
// [fact, dim x D] of a star join) addresses `src`; JOIN_NO_ROW (the NULL-extended side) gives NULL.  dst_null may be nullptr when no
// element can be NULL
__global__ void k_join_rows_gather(DevCol src, const uint32_t* tuples, int width, int which, uint32_t n, int eb, uint8_t* dst, uint8_t* dst_null) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t r = tuples[(size_t)width * i + which];
        const bool isnull = r == JOIN_NO_ROW || elem_is_null(src, r);
        if (dst_null) dst_null[i] = isnull ? 1 : 0;
        const uint8_t* s = (const uint8_t*)src.values + (size_t)r * eb;
        uint8_t* d = dst + (size_t)i * eb;
        if (isnull) { for (int b = 0; b < eb; b++) d[b] = 0; continue; }
        switch (eb) {
            case 1: *d = *s; break;
            case 4: *(uint32_t*)d = *(const uint32_t*)s; break;
            case 8: *(uint64_t*)d = *(const uint64_t*)s; break;
            default: for (int b = 0; b < eb; b++) d[b] = s[b]; break;
        }
    }
}

// K4 build: insert (cast key image, row) of every non-NULL build row (Joiner::construct_hash_map, joiner.cpp:624-631)
__global__ void k_join_build(DevCol key, int from_prim, int cast_to, int64_t nrows, uint64_t* keys, uint32_t* rows, uint32_t cap_mask) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        if (elem_is_null(key, r)) continue;
        const uint64_t img = cast_prim(load_elem(key, r), from_prim, cast_to);
        uint32_t slot = hash_key1(img) & cap_mask;
        for (;;) {
            if (atomicCAS(rows + slot, 0xFFFFFFFFu, (uint32_t)r) == 0xFFFFFFFFu) { keys[slot] = img; break; }
            slot = (slot + 1) & cap_mask;
        }
    }
}

// ---- FK -> PK fast path (see JoinFast in api_state.h) ----
__global__ void k_join_minmax(DevCol key, int from_prim, int cast_to, int64_t nrows, uint64_t bias, uint64_t* mm) {
    uint64_t lo = ~0ull, hi = 0;
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r0 < nrows; r0 += 4 * T) {   // four independent loads in flight per thread
        uint64_t v[4]; bool ok[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t r = r0 + u * T;
            ok[u] = r < nrows && !elem_is_null(key, r);
            v[u] = ok[u] ? load_elem(key, r) : 0;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if (!ok[u]) continue;
            const uint64_t x = cast_prim(v[u], from_prim, cast_to) ^ bias;
            lo = x < lo ? x : lo; hi = x > hi ? x : hi;
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const uint64_t l2 = __shfl_xor_sync(0xFFFFFFFFu, lo, d), h2 = __shfl_xor_sync(0xFFFFFFFFu, hi, d);
        lo = l2 < lo ? l2 : lo; hi = h2 > hi ? h2 : hi;
    }
    if ((threadIdx.x & 31) == 0) { atomicMin((unsigned long long*)mm, (unsigned long long)lo); atomicMax((unsigned long long*)(mm + 1), (unsigned long long)hi); }
}
__global__ void k_join_build_fast(DevCol key, int from_prim, int cast_to, int64_t nrows, JoinFast jf, uint32_t* dense_w, uint64_t* packed_w, uint32_t* dup_flag) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        if (elem_is_null(key, r)) continue;   // a NULL key never matches
        const uint64_t img = cast_prim(load_elem(key, r), from_prim, cast_to);
        if (jf.mode == 1) {
            const uint64_t off = (img ^ jf.bias) - jf.dense_min;
            if (off >= jf.dense_size) { atomicExch(dup_flag + 2, 1u); continue; }   // outside the range learned from an earlier run of the plan: the host rebuilds
            if (atomicExch(dense_w + off, (uint32_t)r) != 0xFFFFFFFFu) atomicExch(dup_flag, 1u);
        } else {
            const uint32_t k32 = (uint32_t)img;
            const uint64_t v = ((uint64_t)k32 << 32) | (uint32_t)r;
            uint32_t slot = (k32 * 0x9E3779B1u) & jf.packed_mask;
            for (;;) {
                const uint64_t old = atomicCAS((unsigned long long*)(packed_w + slot), ~0ull, (unsigned long long)v);
                if (old == ~0ull) break;
                if ((uint32_t)(old >> 32) == k32) { atomicExch(dup_flag, 1u); break; }   // duplicate key: not a PK
                slot = (slot + 1) & jf.packed_mask;
            }
        }
    }
}
__device__ __forceinline__ uint32_t join_lookup(const JoinFast& jf, uint64_t img) {
    if (jf.mode == 1) {
        const uint64_t off = (img ^ jf.bias) - jf.dense_min;
        return off < jf.dense_size ? __ldg(jf.dense + off) : 0xFFFFFFFFu;
    }
    const uint32_t k32 = (uint32_t)img;
    uint32_t slot = (k32 * 0x9E3779B1u) & jf.packed_mask;
    for (;;) {
        const uint64_t v = __ldg((const unsigned long long*)(jf.packed + slot));
        if (v == ~0ull) return 0xFFFFFFFFu;
        if ((uint32_t)(v >> 32) == k32) return (uint32_t)v;
        slot = (slot + 1) & jf.packed_mask;
    }
}
// gather the build-side columns to probe-row alignment; four independent rows per thread keep the random
// lookups and gathers in flight together
__global__ void __launch_bounds__(256) k_join_gather(DevCol pk, int from_prim, int cast_to, int64_t nrows, JoinFast jf, GatherCols gc, uint32_t* miss_flag) {
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    bool miss = false;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; base < nrows; base += 4 * T) {
        uint32_t br[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t r = base + u * T;
            br[u] = 0xFFFFFFFEu;   // beyond the batch
            if (r < nrows) br[u] = elem_is_null(pk, r) ? 0xFFFFFFFFu : join_lookup(jf, cast_prim(load_elem(pk, r), from_prim, cast_to));
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int64_t r = base + u * T;
            if (br[u] == 0xFFFFFFFEu) continue;
            if (br[u] == 0xFFFFFFFFu) { miss = true; continue; }
            for (int c = 0; c < gc.n; c++) {
                if (gc.elem[c] == 8) ((uint64_t*)gc.dst[c])[r] = __ldg((const unsigned long long*)gc.src[c] + br[u]);
                else if (gc.elem[c] == 4) ((uint32_t*)gc.dst[c])[r] = __ldg((const uint32_t*)gc.src[c] + br[u]);
                else if (gc.elem[c] == 16) ((uint4*)gc.dst[c])[r] = __ldg((const uint4*)gc.src[c] + br[u]);   // a MERGE_AGG's AVG {sum, count} blob
                else gc.dst[c][r] = __ldg(gc.src[c] + br[u]);
            }
        }
    }
    if (__any_sync(0xFFFFFFFFu, miss) && (threadIdx.x & 31) == 0) atomicExch(miss_flag, 1u);
}
// K4 fused probe (JoinProbe): compose the grouped-by build attribute onto the key index built by k_join_build_fast
__global__ void k_join_compose(JoinFast jf, const uint32_t* attr_by_row, uint32_t* attr_of_key, uint64_t* packed_attr, uint32_t* bad_flag) {
    const uint64_t n = jf.mode == 1 ? jf.dense_size : (uint64_t)jf.packed_mask + 1;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (jf.mode == 1) {
            const uint32_t r = jf.dense[i];
            attr_of_key[i] = r == 0xFFFFFFFFu ? 0u : __ldg(attr_by_row + r);
        } else {
            const uint64_t e = jf.packed[i];
            uint64_t o = ~0ull;
            if (e != ~0ull) {
                o = (e & 0xFFFFFFFF00000000ull) | __ldg(attr_by_row + (uint32_t)e);
                if (o == ~0ull) atomicExch(bad_flag, 1u);   // (key, attribute) = (0xFFFFFFFF, 0xFFFFFFFF) would read as a free slot
            }
            packed_attr[i] = o;
        }
    }
}

// ---- K4 star join (PK_STAR_AGG): one fact table INNER-joined to up to four dimensions ----
// Build time: the conjuncts over one dimension alone, once per dimension row.  A row's build key is valid when the key is not NULL and the
// conjunction is TRUE: this bitmap (beside the column's own) is the key's validity for k_join_build_fast / k_join_build, which skip NULL keys.
// The two-table join runs it over a child's own filter: the build side's (with `dropped`: a row whose conjunction is not TRUE, whatever its
// key, is marked 2 in matched[]) and each probe batch's.  The program reads the row both as the probe row and as the build row.
__global__ void __launch_bounds__(256) k_star_dim_filter(const __grid_constant__ StarFilter a, uint32_t* keybits, uint8_t* dropped) {
    const int lane = threadIdx.x & 31;
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    for (int64_t w0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); w0 < a.nrows; w0 += T) {   // (warp-uniform: one bitmap word per warp and pass)
        const int64_t r = w0 + lane;
        bool ok = r < a.nrows && !elem_is_null(a.cols[a.key_col], r);
        if ((ok || (dropped && r < a.nrows)) && a.prog.n_instr > 0) {
            uint64_t out[1]; uint32_t out_null;
            run_program(a.prog, a.cols, r, out, out_null, r);
            const bool pass = !(out_null & 1u) && out[0] != 0;
            ok = ok && pass;
            if (dropped && !pass) dropped[r] = 2;
        }
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, ok);
        if (lane == 0) keybits[w0 >> 5] = m;
    }
}
// four consecutive foreign keys [r0, r0 + 4) as canonical images: one 128-bit load (4-byte keys) or two (8-byte keys) when the chunk is 32-byte
// aligned and the four rows exist
__device__ __forceinline__ void load_quad(const DevCol& c, int64_t r0, int64_t nrows, bool vec, uint64_t (&v)[4]) {
    if (vec && r0 + 4 <= nrows && (c.stype == ST_I32 || c.stype == ST_U32)) {
        const uint4 q = __ldg((const uint4*)((const uint32_t*)c.values + r0));
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int u = 0; u < 4; u++) v[u] = narrow_prim(c.stype == ST_I32 ? (uint64_t)(int64_t)(int32_t)w[u] : (uint64_t)w[u], c.prim);
        return;
    }
    if (vec && r0 + 4 <= nrows && (c.stype == ST_I64 || c.stype == ST_U64)) {
        const ulonglong2 a = __ldg((const ulonglong2*)((const unsigned long long*)c.values + r0));
        const ulonglong2 b = __ldg((const ulonglong2*)((const unsigned long long*)c.values + r0 + 2));
        v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
        return;
    }
#pragma unroll
    for (int u = 0; u < 4; u++) v[u] = r0 + u < nrows ? load_elem(c, r0 + u) : 0;
}
// Probe: one pass over a chunk's fact rows.  A row survives when every dimension with unique keys has a partner (a NULL foreign key has none:
// one L2-resident index read per dimension).  Survivors leave as row-id tuples [fact row, dim row x D] in any order, compacted with warp
// ballots and one cursor atomic per warp; the slots of dimensions with duplicate keys are filled by k_star_expand.
__global__ void __launch_bounds__(256) k_star_probe(const __grid_constant__ StarProbe a, uint32_t* out, uint32_t* cursor) {
    const int lane = threadIdx.x & 31;
    const int64_t T = (int64_t)gridDim.x * blockDim.x;
    const int64_t nq = (a.nrows + 3) / 4;
    for (int64_t q0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); q0 < nq; q0 += T) {   // (warp-uniform trip count: the ballots below)
        const int64_t r0 = (q0 + lane) * 4;
        uint32_t br[4][4];
        // every lookup is issued before any result is tested: up to 16 independent index reads in flight per thread
#pragma unroll
        for (int d = 0; d < 4; d++) {
            if (d >= a.n) break;
            const StarLookup& L = a.d[d];
            uint64_t v[4];
            load_quad(L.fk, r0, a.nrows, a.vec != 0, v);
#pragma unroll
            for (int u = 0; u < 4; u++)
                br[u][d] = r0 + u < a.nrows && !elem_is_null(L.fk, r0 + u) ? join_lookup(L.jf, cast_prim(v[u], L.from_prim, L.cast_prim)) : JOIN_NO_ROW;
        }
        uint32_t live = 0;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            bool ok = r0 + u < a.nrows;
#pragma unroll
            for (int d = 0; d < 4; d++) if (d < a.n) ok = ok && br[u][d] != JOIN_NO_ROW;
            if (ok) live |= 1u << u;
        }
        uint32_t b[4]; uint32_t total = 0;
#pragma unroll
        for (int u = 0; u < 4; u++) { b[u] = __ballot_sync(0xFFFFFFFFu, (live >> u) & 1u); total += (uint32_t)__popc(b[u]); }
        if (total == 0) continue;
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(cursor, total);
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if ((live >> u) & 1u) {
                uint32_t* t = out + (size_t)a.width * (base + (uint32_t)__popc(b[u] & lt));
                t[0] = (uint32_t)(r0 + u);
#pragma unroll
                for (int d = 0; d < 4; d++) if (d < a.n) t[a.d[d].slot] = br[u][d];
            }
            base += (uint32_t)__popc(b[u]);
        }
    }
}
// A dimension with duplicate keys: every tuple becomes one tuple per matching row of the dimension's multimap (k_join_build), or none.
// Past `cap` only the count goes on: the host grows the buffer to the count and runs the pass again.
__global__ void __launch_bounds__(256) k_star_expand(DevCol fk, int from_prim, int cast_to, const uint64_t* keys, const uint32_t* rows, uint32_t cap_mask,
                                                     const uint32_t* in, uint32_t n_in, int width, int slot, uint32_t* out, uint32_t cap, uint32_t* cursor) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_in; i += gridDim.x * blockDim.x) {
        const uint32_t* t = in + (size_t)width * i;
        const uint32_t f = t[0];
        if (elem_is_null(fk, f)) continue;
        const uint64_t img = cast_prim(load_elem(fk, f), from_prim, cast_to);
        for (uint32_t h = hash_key1(img) & cap_mask;; h = (h + 1) & cap_mask) {
            const uint32_t br = rows[h];
            if (br == 0xFFFFFFFFu) break;
            if (keys[h] != img) continue;
            const uint32_t pos = atomicAdd(cursor, 1u);
            if (pos >= cap) continue;
            uint32_t* o = out + (size_t)width * pos;
            for (int k = 0; k < width; k++) o[k] = t[k];
            o[slot] = br;
        }
    }
}

}  // namespace bk

// every plan column of the joined row: the build sides' retained columns and the probe batch's (nullptr: the outer-join tail, whose
// probe-side columns are never read — row = -1 is NULL)
static std::vector<DevCol> join_cols(const bkgpu_plan* p, const DevCol* probe_cols) {
    const Compiled& c = p->c;
    std::vector<DevCol> all(c.cols.size());
    for (size_t i = 0; i < c.cols.size(); i++) {
        all[i].stype = prim_storage(c.cols[i].prim); all[i].prim = c.cols[i].prim;
        if (c.col_side[i] > 0) all[i] = store_col(p->join.side[c.col_side[i] - 1].store, i);
    }
    if (probe_cols) for (size_t w = 0; w < p->join.probe_map.size(); w++) all[(size_t)p->join.probe_map[w]] = probe_cols[w];
    return all;
}

// a 4-byte device counter, read once the stream has reached it
static int read_u32(bkgpu_plan* p, const uint32_t* dev, uint32_t* out) {
    CK(p, cudaMemcpyAsync(out, dev, 4, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    return BKGPU_OK;
}
// a pass whose output can outgrow its buffer: `run(cap)` sizes the buffer for `cap` items and launches the pass, which writes at most
// `cap` of them and counts all of them in `cursor`; a pass that found more is rerun once, with the buffer grown to the count
template <class Run>
static int run_counted(bkgpu_plan* p, uint64_t cap, const uint32_t* cursor, uint32_t* found, Run run) {
    for (int attempt = 0; attempt < 2; attempt++) {
        int rc;
        if ((rc = run(cap)) || (rc = read_u32(p, cursor, found))) return rc;
        if (*found <= cap) break;
        cap = *found;
    }
    return BKGPU_OK;
}

JoinArgs join_args(const bkgpu_plan* p, bool tail) {
    const Compiled& c = p->c;
    const JoinSide& s = p->join.side[0];
    JoinArgs a; memset(&a, 0, sizeof a);
    a.enabled = 1; a.keys = s.jt_keys; a.rows = s.jt_rows; a.cap_mask = s.jt_mask;
    a.probe_col = c.probe_key_col; a.probe_prim = c.cols[(size_t)c.probe_key_col].prim; a.cast_prim = c.join_key_prim;
    a.join_type = c.join_type; a.matched = c.join_type == BK_INNER_JOIN ? nullptr : p->join.matched; a.n_build = s.store.rows;
    a.tail = tail ? 1 : 0;
    return a;
}

// ---- retain the build (outer / driver) table, build its indexes at the first probe batch ----
// `side`: the Compiled::col_side value of this table's columns (1 for the two-table join, 1 + d for dimension d of a star join)
static int join_retain_build(bkgpu_plan* p, int side, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    const Compiled& c = p->c;
    JoinSide& s = p->join.side[side - 1];
    if (p->join.built) return p->fail(BKGPU_ESTATE, "build-side rows arrived after probing started (the reference fetches the whole driver table first, join_node.cpp:920-1022)");
    const size_t nc = c.cols.size();
    std::vector<ColRef> want; std::vector<int> idx;
    for (size_t i = 0; i < nc; i++) if (c.col_side[i] == side) { want.push_back(c.cols[i]); idx.push_back((int)i); }
    std::vector<const bkgpu_column*> bound;
    int rc = bind_columns(p, want, cols, ncols, nrows, bound);
    if (rc) return rc;
    if (s.store.rows + nrows > 0xFFFFFFF0ll) return p->fail(BKGPU_EUNSUPPORTED, "build side larger than 2^32 rows");
    if ((rc = store_retain(p, s.store, s.store.rows + nrows))) return rc;
    for (size_t w = 0; w < want.size(); w++) {
        if ((rc = store_append(p, s.store, (size_t)idx[w], *bound[w], nrows, on_device))) return rc;
        if (on_device) p->stats.kernel_launches++;   // (the unpack kernel)
    }
    s.store.rows += nrows;
    return BKGPU_OK;
}

// Fused probe (JoinProbe in agg.h): usable when the only build-side column the aggregate reads is its 4-byte GROUP BY
// key and the probe key is a 32-bit integer column whose cast to the comparison type keeps the canonical image.
static int join_compose_probe(bkgpu_plan* p, uint32_t* flag) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    const JoinSide& s = j.side[0];
    j.jp = JoinProbe{};
    if (!c.jfast || !c.jfast->has_direct || c.jfast->direct.n_keys != 1) return BKGPU_OK;
    const Compiled& f = *c.jfast;
    const size_t kpos = (size_t)f.direct.n_terms;
    int attr_main = -1;
    for (size_t i = 0; i < f.direct_cols.size(); i++) {
        const int m = c.jfast_of_main[(size_t)f.direct_cols[i]];
        if (c.col_side[(size_t)m] != 1) continue;
        if (i != kpos) return BKGPU_OK;   // a predicate or an aggregate argument comes from the build side: gather path
        attr_main = m;
    }
    if (attr_main < 0) return BKGPU_OK;
    const int ast = prim_storage(c.cols[(size_t)attr_main].prim);
    if ((ast != ST_I32 && ast != ST_U32) || (c.cols[(size_t)attr_main].prim != BK_INT32 && c.cols[(size_t)attr_main].prim != BK_UINT32)) return BKGPU_OK;
    const int pp = c.cols[(size_t)c.probe_key_col].prim, ct = c.join_key_prim;
    const bool ident = (pp == BK_INT32 && (ct == BK_INT32 || ct == BK_INT64)) || (pp == BK_UINT32 && (ct == BK_UINT32 || ct == BK_UINT64 || ct == BK_INT64));
    if (!ident) return BKGPU_OK;
    int rc;
    JoinProbe jp{};
    jp.mode = s.jf.mode; jp.key_signed = pp == BK_INT32 ? 1 : 0;
    jp.dense_min = s.jf.dense_min; jp.dense_size = s.jf.dense_size; jp.bias = s.jf.bias; jp.packed_mask = s.jf.packed_mask;
    if (jp.mode == 1) {
        if ((rc = ensure_buf(p, (void**)&j.jp_attr, &j.jp_attr_cap, (size_t)jp.dense_size * 4))) return rc;
        jp.attr = j.jp_attr;
        jp.present = (uint64_t)s.store.rows == jp.dense_size ? nullptr : s.jf.dense;   // unique, NULL-free keys filling the range: every key exists
    } else {
        if ((rc = ensure_buf(p, (void**)&j.jp_packed, &j.jp_packed_cap, ((size_t)jp.packed_mask + 1) * 8))) return rc;
        jp.packed = j.jp_packed;
    }
    CK(p, cudaMemsetAsync(flag, 0, 4, p->stream));
    const uint64_t n_idx = s.jf.mode == 1 ? s.jf.dense_size : (uint64_t)s.jf.packed_mask + 1;
    k_join_compose<<<grid_for((int64_t)n_idx, p->sm_count, 16), 256, 0, p->stream>>>(s.jf, (const uint32_t*)s.store.cols[(size_t)attr_main].vals, j.jp_attr, j.jp_packed, flag);
    CK(p, cudaGetLastError());
    p->stats.kernel_launches++;
    j.jp = jp; j.jp_key_pos = (int)kpos;   // (the caller drops it again when `flag` comes back set)
    return BKGPU_OK;
}

// validity bitmaps of the side's retained columns that some batch delivered NULLs for (store_col reads no bitmap of the others)
static int join_pack_validity(bkgpu_plan* p, JoinSide& s) {
    int rc;
    DevCol d;
    for (size_t i = 0; i < s.store.cols.size(); i++) {
        if (!s.store.cols[i].nullable) continue;
        if ((rc = store_pack(p, s.store, i, s.store.rows, 16, nullptr, &d))) return rc;
        p->stats.kernel_launches++;
    }
    return BKGPU_OK;
}

// The unique-key index of side `s` (FK -> PK fast path): a dense array when the key range is small, else a packed table for keys of at most
// 32 bits.  s.jf.mode stays 0 when neither fits or a key repeats.  `compose`: the two-table join's fused probe is composed behind the build,
// so that its flag comes back in the same round trip.
static int join_build_index(bkgpu_plan* p, JoinSide& s, const DevCol& key, int cast_prim, bool compose) {
    JoinState& j = p->join;
    int rc;
    s.jf = JoinFast{};
    if (s.store.rows <= 0) return BKGPU_OK;
    if ((rc = ensure_buf(p, (void**)&j.cursor, &j.cursor_cap, 64))) return rc;   // (the gather's misses, the star probe's survivors)
    bool retry_measured = false;
again:
    const int cls = host_prim_class(cast_prim);
    const uint64_t bias = cls == VC_I64 ? 0x8000000000000000ull : 0ull;
    if ((rc = ensure_buf(p, (void**)&j.scratch, &j.scratch_cap, 64))) return rc;
    uint64_t* mm = j.scratch; uint32_t* dup = (uint32_t*)(j.scratch + 2);
    // the key range: measured (one pass over the keys + a round trip), or — when this plan has built before — the range it saw then,
    // checked by the build kernel itself (a key outside it raises a flag and the build is redone with a measured range)
    uint64_t h_mm[2];
    bool guessed = s.learned && !retry_measured;
    if (guessed) { h_mm[0] = s.learn_min; h_mm[1] = s.learn_max; }
    else {
        const uint64_t init[2] = {~0ull, 0ull};
        CK(p, cudaMemcpyAsync(mm, init, 16, cudaMemcpyHostToDevice, p->stream));
        k_join_minmax<<<grid_for(s.store.rows, p->sm_count, 8), 256, 0, p->stream>>>(key, key.prim, cast_prim, s.store.rows, bias, mm);
        CK(p, cudaGetLastError());
        CK(p, cudaMemcpyAsync(h_mm, mm, 16, cudaMemcpyDeviceToHost, p->stream));
        CK(p, cudaStreamSynchronize(p->stream));
        p->stats.kernel_launches++;
    }
    JoinFast jf{}; jf.bias = bias;
    const uint64_t range = h_mm[1] >= h_mm[0] ? h_mm[1] - h_mm[0] + 1 : 0;
    const int kb = storage_bytes(prim_storage(cast_prim));
    if (range > 0 && range <= (uint64_t)4 * (uint64_t)s.store.rows + 1024 && range <= (1ull << 30)) {
        jf.mode = 1; jf.dense_min = h_mm[0]; jf.dense_size = range;
        if ((rc = ensure_buf(p, (void**)&s.jf_dense, &s.jf_dense_cap, (size_t)range * 4))) return rc;
        jf.dense = s.jf_dense;
    } else if (kb <= 4) {
        uint32_t pc = 1024; while ((int64_t)pc < 2 * s.store.rows) pc <<= 1;
        jf.mode = 2; jf.packed_mask = pc - 1;
        if ((rc = ensure_buf(p, (void**)&s.jf_packed, &s.jf_packed_cap, (size_t)pc * 8))) return rc;
        jf.packed = s.jf_packed;
    }
    if (jf.mode) {
        CK(p, cudaMemsetAsync(dup, 0, 12, p->stream));   // [0] duplicate key, [1] fused probe unusable (set by the compose step), [2] key outside the guessed range
        if (jf.mode == 1) CK(p, cudaMemsetAsync(s.jf_dense, 0xFF, jf.dense_size * 4, p->stream));
        else CK(p, cudaMemsetAsync(s.jf_packed, 0xFF, ((size_t)jf.packed_mask + 1) * 8, p->stream));
        k_join_build_fast<<<grid_for(s.store.rows, p->sm_count, 16), 256, 0, p->stream>>>(key, key.prim, cast_prim, s.store.rows, jf, s.jf_dense, s.jf_packed, dup);
        CK(p, cudaGetLastError());
        p->stats.kernel_launches += 1;
        s.jf = jf;
        if (compose && (rc = join_compose_probe(p, dup + 1))) return rc;   // enqueued behind the build: all flags come back in one round trip
        uint32_t h_flags[3] = {0, 0, 0};
        CK(p, cudaMemcpyAsync(h_flags, dup, 12, cudaMemcpyDeviceToHost, p->stream));
        CK(p, cudaStreamSynchronize(p->stream));
        if (h_flags[2] && guessed) { retry_measured = true; goto again; }   // this run's keys left the learned range
        if (h_flags[0]) { s.jf = JoinFast{}; j.jp = JoinProbe{}; }   // duplicate build keys: not a PK, the general probe runs
        else if (h_flags[1]) j.jp = JoinProbe{};
        s.learned = true; s.learn_min = h_mm[0]; s.learn_max = h_mm[1];
    } else if (guessed) { retry_measured = true; goto again; }   // (the learned range no longer fits this row count)
    return BKGPU_OK;
}

static int join_build_table(bkgpu_plan* p) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    JoinSide& s = j.side[0];
    int rc;
    if ((rc = join_pack_validity(p, s))) return rc;
    j.built = true; s.jt_generic = false;   // the multimap of the general probe is built on first use (join_generic_table)
    // ---- FK -> PK fast path: are the build keys unique, and is their range dense or their type <= 32 bits? ----
    s.jf = JoinFast{}; j.jp = JoinProbe{};
    bool build_nulls = false;
    for (const RowStore::Col& col : s.store.cols) if (col.nullable) build_nulls = true;   // gathered columns must be NULL-free
    if (!c.jfast || c.join_type == BK_FULL_JOIN || build_nulls) return BKGPU_OK;
    return join_build_index(p, s, store_col(s.store, (size_t)c.build_key_col), c.join_key_prim, true);
}

// the multimap of side `s` (duplicate build keys, the general probe): open addressing from the cast key image to the build row
static int join_build_multimap(bkgpu_plan* p, JoinSide& s, const DevCol& key, int cast_prim) {
    int rc;
    uint32_t cap = 1024;
    while ((int64_t)cap < 2 * s.store.rows) cap <<= 1;
    dev_free(p, s.jt_keys); dev_free(p, s.jt_rows); s.jt_keys = nullptr; s.jt_rows = nullptr;
    if ((rc = dev_alloc(p, (void**)&s.jt_keys, (size_t)cap * 8))) return rc;
    if ((rc = dev_alloc(p, (void**)&s.jt_rows, (size_t)cap * 4))) return rc;
    s.jt_mask = cap - 1;
    CK(p, cudaMemsetAsync(s.jt_rows, 0xFF, (size_t)cap * 4, p->stream));
    if (s.store.rows > 0) {
        k_join_build<<<grid_for(s.store.rows, p->sm_count, 16), 256, 0, p->stream>>>(key, key.prim, cast_prim, s.store.rows, s.jt_keys, s.jt_rows, s.jt_mask);
        CK(p, cudaGetLastError());
    }
    p->stats.kernel_launches++;
    s.jt_generic = true;
    return BKGPU_OK;
}

// a two-table join child's own filter (Compiled::build_filter / probe_filter) over `nrows` rows of `cols` (every plan column, this child's at
// the rows' start) into *bits: "key not NULL and the conjunction TRUE".  `dropped`: matched[] of the build side, 2 where the conjunction is not TRUE
static int join_child_filter(bkgpu_plan* p, const Program& prog, int key_col, const DevCol* cols, int64_t nrows, uint8_t** bits, size_t* bits_cap, uint8_t* dropped) {
    const Compiled& c = p->c;
    int rc;
    if ((rc = ensure_buf(p, (void**)bits, bits_cap, ((size_t)nrows + 31) / 32 * 4 + 4))) return rc;
    StarFilter f; memset(&f, 0, sizeof f);
    for (size_t i = 0; i < c.cols.size(); i++) f.cols[i] = cols[i];
    f.prog = prog; f.key_col = key_col; f.nrows = nrows;
    if (nrows > 0) {
        k_star_dim_filter<<<grid_for(nrows, p->sm_count, 16), 256, 0, p->stream>>>(f, (uint32_t*)*bits, dropped);
        CK(p, cudaGetLastError());
    }
    p->stats.kernel_launches++;
    return BKGPU_OK;
}

// the general probe's multimap (duplicate build keys, unmatched probe rows): built only when a batch needs it
static int join_generic_table(bkgpu_plan* p) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    JoinSide& s = j.side[0];
    if (s.jt_generic) return BKGPU_OK;
    int rc;
    DevCol key = store_col(s.store, (size_t)c.build_key_col);
    if (c.join_type != BK_INNER_JOIN) {   // one "found a partner" byte per build row
        if ((rc = ensure_buf(p, (void**)&j.matched, &j.matched_cap, (size_t)std::max<int64_t>(s.store.rows, 1)))) return rc;
        CK(p, cudaMemsetAsync(j.matched, 0, (size_t)std::max<int64_t>(s.store.rows, 1), p->stream));
        if (c.n_build_filter > 0) {   // (SEMI / ANTI) a row that fails its own filter is neither in the multimap nor in the tail
            const std::vector<DevCol> all = join_cols(p, nullptr);
            if ((rc = join_child_filter(p, c.build_filter, c.build_key_col, all.data(), s.store.rows, &s.keybits, &s.keybits_cap, j.matched))) return rc;
            key.validity = s.keybits;
        }
    }
    return join_build_multimap(p, s, key, c.join_key_prim);
}

// the probe child's own filter over one batch (`all`: every plan column): its bitmap becomes the probe key's validity for the batch, so a row that
// fails it finds no partner, as a row with a NULL key.  Never for FULL, where such a row would still come out NULL-extended.  A row that passes
// has a valid key: every row the aggregate or the sink sees reads the key column as before.
static int join_probe_filter(bkgpu_plan* p, std::vector<DevCol>& all, int64_t nrows) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    if (c.n_probe_filter == 0) return BKGPU_OK;
    const int rc = join_child_filter(p, c.probe_filter, c.probe_key_col, all.data(), nrows, &j.probe_bits, &j.probe_bits_cap, nullptr);
    all[(size_t)c.probe_key_col].validity = j.probe_bits;
    return rc;
}

static int join_probe_batch(bkgpu_plan* p, const DevCol* probe_cols, int64_t nrows, int64_t, bool) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    const JoinSide& s = j.side[0];
    std::vector<DevCol> all = join_cols(p, probe_cols);
    // ---- FK -> PK fast path: gather the build columns next to the probe rows, then the ordinary (lean) aggregate ----
    if (s.jf.mode != 0 && j.jp.mode != 0 && c.jfast && !p->agg.env.force_generic && !j.no_fused_probe) {
        // ---- fused probe: the lean aggregate reads the foreign key and looks the group key up itself ----
        const Compiled& f = *c.jfast;
        std::vector<DevCol> fc(f.cols.size());
        const int key_fcol = f.direct_cols[(size_t)j.jp_key_pos];
        bool vec_ok = true;
        for (size_t i = 0; i < f.cols.size(); i++) {
            fc[i] = (int)i == key_fcol ? all[(size_t)c.probe_key_col] : all[(size_t)c.jfast_of_main[i]];
            if (((uintptr_t)fc[i].values & 31) != 0) vec_ok = false;
        }
        const int rc = launch_agg_batch(p, f, fc.data(), nrows, vec_ok, &j.jp);
        if (rc <= 0) return rc;   // launched (0) or failed (< 0); +1: this batch does not fit the lean kernel
    }
    if (s.jf.mode != 0 && c.jfast && !p->agg.env.force_generic) {
        const Compiled& f = *c.jfast;
        const int64_t chunk = 16 << 20;   // the gathered chunk is re-read immediately: keep it L2-sized
        for (int64_t off = 0; off < nrows; off += chunk) {
            const int64_t n = std::min(chunk, nrows - off);
            GatherCols gc{}; std::vector<DevCol> fc(f.cols.size());
            int rc;
            for (size_t i = 0; i < f.cols.size(); i++) {
                const size_t m = (size_t)c.jfast_of_main[i];
                if (c.col_side[m] != 1) { fc[i] = col_at(all[m], off); continue; }
                if ((rc = store_reserve(p, j.chunk, m, chunk, chunk, false))) return rc;
                uint8_t* dst = j.chunk.cols[m].vals;
                gc.src[gc.n] = s.store.cols[m].vals; gc.dst[gc.n] = dst; gc.elem[gc.n] = storage_bytes(all[m].stype); gc.n++;
                fc[i] = all[m]; fc[i].values = dst; fc[i].validity = nullptr;
            }
            CK(p, cudaMemsetAsync(j.cursor, 0, 4, p->stream));
            k_join_gather<<<grid_for((n + 3) / 4, p->sm_count, 8), 256, 0, p->stream>>>(col_at(all[(size_t)c.probe_key_col], off), c.cols[(size_t)c.probe_key_col].prim,
                                                                                       c.join_key_prim, n, s.jf, gc, j.cursor);
            CK(p, cudaGetLastError());
            p->stats.kernel_launches++;
            uint32_t miss = 0;
            if ((rc = read_u32(p, j.cursor, &miss))) return rc;
            if (miss) {   // some probe row has no partner (or a NULL key): this chunk takes the general probe
                std::vector<DevCol> sl(all);
                for (size_t i = 0; i < sl.size(); i++) if (c.col_side[i] == 0) sl[i] = col_at(all[i], off);
                if ((rc = join_generic_table(p))) return rc;
                if ((rc = launch_agg_batch(p, c, sl.data(), n, false))) return rc;
            } else {
                bool vec_ok = true;
                for (auto& d : fc) if (((uintptr_t)d.values & 31) != 0) vec_ok = false;
                if ((rc = launch_agg_batch(p, f, fc.data(), n, vec_ok))) return rc;
            }
        }
        return BKGPU_OK;
    }
    { int rc; if ((rc = join_generic_table(p)) || (rc = join_probe_filter(p, all, nrows))) return rc; }
    return launch_agg_batch(p, c, all.data(), nrows, false);
}

// the (probe row, build row) pairs of `n_probe` probe rows (`all`: every plan column, the probe side's at the rows' start), or of the
// outer-join tail, into j.pairs; *found = their number
static int join_pairs(bkgpu_plan* p, const std::vector<DevCol>& all, int64_t n_probe, bool tail, uint32_t* found) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    int rc;
    AggArgs a; memset(&a, 0, sizeof a);
    a.plan = c.ap; a.prog = c.prog; a.nrows = n_probe;
    const int ncols = (int)c.cols.size();
    for (int i = 0; i < ncols; i++) a.cols[i] = all[(size_t)i];
    a.n_cols = ncols;
    a.join = join_args(p, tail);
    if ((rc = ensure_buf(p, (void**)&j.cursor, &j.cursor_cap, 64))) return rc;
    *found = 0;
    return run_counted(p, (uint64_t)std::max<int64_t>(tail ? j.side[0].store.rows : n_probe, 1 << 12), j.cursor, found, [&](uint64_t want) -> int {
        if (want > 0x7FFFFFF0ull) return p->fail(BKGPU_ETOOBIG, "a probe batch joins to more than 2^31 rows: push smaller batches");
        int r;
        if ((r = ensure_buf(p, (void**)&j.pairs, &j.pairs_cap, (size_t)want * 8))) return r;
        CK(p, cudaMemsetAsync(j.cursor, 0, 4, p->stream));
        // (a rerun of a LEFT / FULL batch sets the same matched[] flags again: they only ever go from 0 to 1; a 2 is never in the multimap)
        CK(p, launch_join_pairs(a, j.pairs, (uint32_t)want, j.cursor, p->sm_count, p->stream));
        p->stats.kernel_launches++;
        return BKGPU_OK;
    });
}

// ---- a JOIN that returns rows (PK_JOIN): pairs -> gather -> the sink fragment (p->post) ----
static int join_rows_emit(bkgpu_plan* p, const std::vector<DevCol>& all, int64_t n_probe, bool tail) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    int rc;
    uint32_t found = 0;
    rc = join_pairs(p, all, n_probe, tail, &found);
    if (rc || !found) return rc;
    rc = sort_feed(p->post, found, std::max<int64_t>((int64_t)found + found / 4, 1 << 16), 16, &p->stats, [&](RowStore& in) {
        for (size_t k = 0; k < in.cols.size(); k++) {   // sink column k = output column k = device column k of the join (plan.cpp::lower_join_rows)
            const RowStore::Col& d = in.cols[k];
            k_join_rows_gather<<<grid_for(found, p->sm_count, 16), 256, 0, p->stream>>>(all[k], j.pairs, 2, c.col_side[k] == 1 ? 1 : 0, found,
                                                                                        storage_bytes(prim_storage(d.prim)), d.vals, d.nulls);
            CK(p, cudaGetLastError());
        }
        return BKGPU_OK;
    });
    if (rc) return rc;
    p->stats.kernel_launches += 2 * (int64_t)c.post->cols.size();
    CK(p, cudaStreamSynchronize(p->stream));   // the gather buffers are reused by the next batch
    return BKGPU_OK;
}
static int join_rows_batch(bkgpu_plan* p, const DevCol* probe_cols, int64_t nrows, int64_t, bool) {
    int rc;
    std::vector<DevCol> all = join_cols(p, probe_cols);
    if ((rc = join_generic_table(p)) || (rc = join_probe_filter(p, all, nrows))) return rc;
    return join_rows_emit(p, all, nrows, false);
}

// ---- FULL join under an aggregate (PK_JOIN_AGG): pairs -> gather -> the aggregate over the joined row (Compiled::jfast, whose predicate is
// the filter above the join).  Never the FK -> PK path: that assumes exactly one partner per probe row. ----
// the pairs of `n_probe` probe rows (or of the tail), every column jfast reads gathered from its pair (NULL on the side a pair lacks), the aggregate
static int full_join_agg(bkgpu_plan* p, const std::vector<DevCol>& all, int64_t n_probe, bool tail) {
    const Compiled& c = p->c;
    const Compiled& f = *c.jfast;
    JoinState& j = p->join;
    uint32_t found = 0;
    int rc = join_pairs(p, all, n_probe, tail, &found);
    if (rc || !found) return rc;
    std::vector<DevCol> fc(f.cols.size());
    for (size_t i = 0; i < f.cols.size(); i++) {
        const size_t m = (size_t)c.jfast_of_main[i];
        if ((rc = store_reserve(p, j.chunk, m, found, found, true))) return rc;
        const RowStore::Col& g = j.chunk.cols[m];
        k_join_rows_gather<<<grid_for(found, p->sm_count, 16), 256, 0, p->stream>>>(all[m], j.pairs, 2, c.col_side[m] == 1 ? 1 : 0, found, storage_bytes(all[m].stype), g.vals, g.nulls);
        CK(p, cudaGetLastError());
        DevCol packed;
        if ((rc = store_pack(p, j.chunk, m, found, 16, nullptr, &packed))) return rc;
        p->stats.kernel_launches += 2;
        fc[i] = all[m]; fc[i].values = g.vals; fc[i].validity = packed.validity;
    }
    return launch_agg_batch(p, f, fc.data(), found, true);
}
static int full_join_probe_batch(bkgpu_plan* p, const DevCol* probe_cols, int64_t nrows, int64_t, bool) {
    const Compiled& c = p->c;
    int rc;
    if ((rc = join_generic_table(p))) return rc;
    const std::vector<DevCol> all = join_cols(p, probe_cols);
    const int64_t chunk = 16 << 20;   // bounds the pairs and the gathered chunk
    for (int64_t off = 0; off < nrows; off += chunk) {
        std::vector<DevCol> sl(all);
        for (size_t i = 0; i < sl.size(); i++) if (c.col_side[i] == 0) sl[i] = col_at(all[i], off);
        if ((rc = full_join_agg(p, sl, std::min(chunk, nrows - off), false))) return rc;
    }
    return BKGPU_OK;
}

// LEFT / SEMI / ANTI_SEMI / FULL: once every probe batch has run, the preserved (build) side's rows the join type asks for go through the
// aggregate (PK_JOIN_AGG) or the sink (PK_JOIN) — unmatched rows NULL-extended (LEFT, FULL), matched rows (SEMI), unmatched rows (ANTI_SEMI);
// join_node.cpp:1200-1276
int join_tail(bkgpu_plan* p) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    if (c.join_type == BK_INNER_JOIN || j.side[0].store.rows == 0) return BKGPU_OK;
    int rc;
    if (!j.built && (rc = join_build_table(p))) return rc;
    if ((rc = join_generic_table(p))) return rc;
    const std::vector<DevCol> all = join_cols(p, nullptr);
    if (c.kind == PK_JOIN) return join_rows_emit(p, all, 0, true);
    if (c.join_type == BK_FULL_JOIN) return full_join_agg(p, all, 0, true);
    j.tail_launch = true;
    rc = launch_agg_batch(p, c, all.data(), j.side[0].store.rows, false);
    j.tail_launch = false;
    return rc;
}

// ---- star join (PK_STAR_AGG): every dimension is retained and indexed before the first fact batch ----
static int star_build(bkgpu_plan* p) {
    const Compiled& c = p->c;
    p->join.built = true;
    int rc;
    for (size_t d = 0; d < c.dims.size(); d++) {
        JoinSide& s = p->join.side[d];
        const StarDim& sd = c.dims[d];
        if ((rc = join_pack_validity(p, s))) return rc;
        s.jt_generic = false; s.jf = JoinFast{};
        if (s.store.rows == 0) continue;
        DevCol key = store_col(s.store, (size_t)sd.key_col);
        if (sd.n_filter > 0) {   // the build key's validity: the key is not NULL and the dimension's own conjuncts are TRUE
            if ((rc = ensure_buf(p, (void**)&s.keybits, &s.keybits_cap, ((size_t)s.store.rows + 31) / 32 * 4))) return rc;
            StarFilter f; memset(&f, 0, sizeof f);
            for (size_t i = 0; i < c.cols.size(); i++) if (c.col_side[i] == 1 + (int)d) f.cols[i] = store_col(s.store, i);
            f.prog = sd.filter; f.key_col = sd.key_col; f.nrows = s.store.rows;
            k_star_dim_filter<<<grid_for(s.store.rows, p->sm_count, 16), 256, 0, p->stream>>>(f, (uint32_t*)s.keybits, nullptr);
            CK(p, cudaGetLastError());
            p->stats.kernel_launches++;
            key.validity = s.keybits;
        }
        // unique keys: the dense or packed index; duplicate keys (or 64-bit keys over a wide range): the multimap
        if ((rc = join_build_index(p, s, key, sd.cast_prim, false))) return rc;
        if (s.jf.mode == 0 && (rc = join_build_multimap(p, s, key, sd.cast_prim))) return rc;
    }
    return BKGPU_OK;
}

// the tuple buffer `k` with room for `n` tuples of `w` row ids
static int star_tuples(bkgpu_plan* p, int k, uint64_t n, int w) {
    if (n * (uint64_t)w > 0xFFFFFFF0ull) return p->fail(BKGPU_ETOOBIG, "a star join chunk joins to more than 2^32 row ids: push smaller batches");
    return ensure_buf(p, (void**)&p->join.tuples[k], &p->join.tuples_cap[k], (size_t)std::max<uint64_t>(n, 1) * (size_t)w * 4);
}

// A fact batch, chunk by chunk: k_star_probe keeps the rows with a partner in every dimension of unique keys, each dimension with duplicate
// keys expands the survivors (k_star_expand), the referenced columns are gathered side by side, and the aggregate runs over them as the
// virtual joined tuple (Compiled::jfast: the lean kernel when the shape fits).
static int star_probe_batch(bkgpu_plan* p, const DevCol* fact_cols, int64_t nrows, int64_t, bool vec_ok) {
    const Compiled& c = p->c;
    const Compiled& f = *c.jfast;
    JoinState& j = p->join;
    const int D = (int)c.dims.size(), W = 1 + D;
    for (int d = 0; d < D; d++) if (j.side[d].store.rows == 0) return BKGPU_OK;   // an empty dimension: no row joins
    const std::vector<DevCol> all = join_cols(p, fact_cols);
    int rc;
    const int64_t chunk = 16 << 20;
    for (int64_t off = 0; off < nrows; off += chunk) {
        const int64_t n = std::min(chunk, nrows - off);
        StarProbe sp; memset(&sp, 0, sizeof sp);
        sp.width = W; sp.nrows = n; sp.vec = vec_ok ? 1 : 0;
        for (int d = 0; d < D; d++) {
            if (j.side[d].jf.mode == 0) continue;
            const StarDim& sd = c.dims[(size_t)d];
            StarLookup& L = sp.d[sp.n++];
            L.fk = col_at(all[(size_t)sd.fk_col], off); L.from_prim = c.cols[(size_t)sd.fk_col].prim; L.cast_prim = sd.cast_prim; L.slot = 1 + d; L.jf = j.side[d].jf;
        }
        if ((rc = star_tuples(p, 0, (uint64_t)n, W))) return rc;
        CK(p, cudaMemsetAsync(j.cursor, 0, 4, p->stream));
        k_star_probe<<<grid_for((n + 3) / 4, p->sm_count, 8), 256, 0, p->stream>>>(sp, j.tuples[0], j.cursor);   // (four rows per thread)
        CK(p, cudaGetLastError());
        p->stats.kernel_launches++;
        uint32_t found = 0;
        if ((rc = read_u32(p, j.cursor, &found))) return rc;
        int cur = 0;
        for (int d = 0; d < D && found; d++) {   // dimensions with duplicate keys: one expansion pass each
            const JoinSide& s = j.side[d];
            if (s.jf.mode != 0) continue;
            const StarDim& sd = c.dims[(size_t)d];
            const DevCol fk = col_at(all[(size_t)sd.fk_col], off);
            uint32_t got = 0;
            rc = run_counted(p, j.star_expand_cap > 0 ? (uint64_t)j.star_expand_cap : std::max<uint64_t>(2 * (uint64_t)found, 4096), j.cursor, &got,
                             [&](uint64_t cap) -> int {
                int r;
                if ((r = star_tuples(p, 1 - cur, cap, W))) return r;
                CK(p, cudaMemsetAsync(j.cursor, 0, 4, p->stream));
                k_star_expand<<<grid_for(found, p->sm_count, 16), 256, 0, p->stream>>>(fk, c.cols[(size_t)sd.fk_col].prim, sd.cast_prim, s.jt_keys, s.jt_rows, s.jt_mask,
                                                                                       j.tuples[cur], found, W, 1 + d, j.tuples[1 - cur], (uint32_t)cap, j.cursor);
                CK(p, cudaGetLastError());
                p->stats.kernel_launches++;
                return BKGPU_OK;
            });
            if (rc) return rc;
            found = got; cur = 1 - cur;
        }
        if (!found) continue;
        // the joined chunk: every column the aggregate reads, gathered from its tuple's row
        std::vector<DevCol> fc(f.cols.size());
        for (size_t i = 0; i < f.cols.size(); i++) {
            const size_t m = (size_t)c.jfast_of_main[i];
            const int side = c.col_side[m];
            const DevCol src = side == 0 ? col_at(all[m], off) : all[m];
            if ((rc = store_reserve(p, j.chunk, m, found, found, src.validity != nullptr))) return rc;   // NULLs travel along: null bytes, then a bitmap
            const RowStore::Col& g = j.chunk.cols[m];
            fc[i] = src; fc[i].values = g.vals; fc[i].validity = nullptr;
            k_join_rows_gather<<<grid_for(found, p->sm_count, 16), 256, 0, p->stream>>>(src, j.tuples[cur], W, side, found, storage_bytes(src.stype), g.vals,
                                                                                        src.validity ? g.nulls : nullptr);
            CK(p, cudaGetLastError());
            p->stats.kernel_launches++;
            if (src.validity) {
                DevCol packed;
                if ((rc = store_pack(p, j.chunk, m, found, 16, nullptr, &packed))) return rc;
                p->stats.kernel_launches++;
                fc[i].validity = packed.validity;
            }
        }
        if ((rc = launch_agg_batch(p, f, fc.data(), found, true))) return rc;
    }
    return BKGPU_OK;
}

// a batch of a build table — the two-table join's build side, a star join's dimensions — is retained; any other batch is probed
int join_push(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    const bool star = c.kind == PK_STAR_AGG;
    if (j.chunk.cols.empty()) {   // the stores' columns, by plan column: a build side holds its own table's
        store_init(j.chunk, c.cols);
        for (int d = 0; d < 4; d++) {
            store_init(j.side[d].store, c.cols);
            for (size_t i = 0; i < c.cols.size(); i++) if (c.col_side[i] != 1 + d) j.side[d].store.cols[i].prim = -1;
        }
    }
    int side = 0;   // (the Compiled::col_side value of the build table's columns)
    if (!star) { for (int k = 0; k < ncols; k++) if (cols[k].tuple_id == c.build_tuple) side = 1; }
    else for (size_t d = 0; d < c.dims.size() && !side; d++) for (int k = 0; k < ncols; k++) if (cols[k].tuple_id == c.dims[d].tuple_id) side = 1 + (int)d;
    if (side) return join_retain_build(p, side, cols, ncols, nrows, on_device);
    if (!j.built) { int rc = star ? star_build(p) : join_build_table(p); if (rc) return rc; }
    if (j.probe_want.empty()) for (size_t i = 0; i < c.cols.size(); i++) if (c.col_side[i] == 0) { j.probe_want.push_back(c.cols[i]); j.probe_map.push_back((int)i); }
    return feed(p, j.probe_want, cols, ncols, nrows, on_device, star ? star_probe_batch : c.kind == PK_JOIN ? join_rows_batch :
                                                                c.join_type == BK_FULL_JOIN ? full_join_probe_batch : join_probe_batch);
}

void join_reset(bkgpu_plan* p) {
    p->join.built = false;
    for (JoinSide& s : p->join.side) {
        s.store.rows = 0; s.jt_generic = false;
        for (RowStore::Col& col : s.store.cols) col.nullable = false;   // (the previous run's bitmaps are not read again)
    }
}

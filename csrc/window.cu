// window.cu — K6: window functions over stably sorted rows, for sm_90a.
//
// Replaces WindowNode / WindowProcessor / WindowFnCall (src/exec/window_node.cpp, src/expr/window_fn_call.cpp).  The reference splits
// the sorted rows into partitions by comparing encode_exprs_key of the partition expressions of adjacent rows, then either calls each
// function once over the whole partition (NonFrameWindowProcessor) or resets and re-aggregates the frame of every row
// (FrameWindowProcessor): O(partition^2) for the default RANGE UNBOUNDED PRECEDING .. CURRENT ROW frame.  Here, after the sort:
//   k_win_eval    : every partition / order / argument expression of the stage, evaluated per row (the device interpreter) and gathered
//                   into sorted order
//   k_win_flags   : partition starts (key bytes differ) and peer-group starts (MemRowCompare != 0) from adjacent rows
//   k_scan_*      : segmented scans (three launches: tile reduce, a one-CTA scan of the tile aggregates, downsweep), forward or backward:
//                   partition / peer-group start and end indices, running COUNT / SUM / MIN / MAX, DENSE_RANK's count of peer starts
//   k_win_fn      : one pass per function: ranking from the indices, LEAD / LAG / FIRST / LAST / NTH as gathers, aggregates read from
//                   a scan at the frame's end (prefix frames), start (suffix frames) or peer group's end, or — bounded ROWS frames of at
//                   most 4096 rows — summed row by row over the frame in order (no difference of prefix sums: a DOUBLE would cancel)
// Results are written at the row's arrival index (row space), so a later stage's sort permutes them with the scan columns.
#include "window.h"
#include <algorithm>
#include <string.h>
#include "api_state.h"
#include "dev_common.cuh"
#include "interp.cuh"
#include "prims.cuh"

namespace bk {

namespace {

struct EvalArgs { DevCol cols[MAX_COLS]; int32_t n_cols; int64_t nrows; Program prog; };

// output 0 of the program for row perm[i], stored at sorted position i
__global__ void k_win_eval(EvalArgs a, const uint32_t* perm, uint64_t* val, uint8_t* nul) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.nrows; i += (int64_t)gridDim.x * blockDim.x) {
        uint64_t out[8]; uint32_t on = 0;
        run_program(a.prog, a.cols, (int64_t)perm[i], out, on);
        const bool isnull = on & 1u;
        val[i] = isnull ? 0ull : out[0];
        nul[i] = isnull ? 1 : 0;
    }
}

struct KeyCmp { const uint64_t* val[4]; const uint8_t* nul[4]; uint8_t is_f64[4]; int n_part, n_keys; };

// part[i]: row i starts a partition (split_into_partitions: the NULL flag and value bytes of some partition key differ from row i-1)
// peer[i]: row i starts a peer group (a partition start, or MemRowCompare::compare of the order keys != 0: -0.0 and +0.0 compare equal)
__global__ void k_win_flags(KeyCmp k, int64_t n, uint8_t* part, uint8_t* peer) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        bool pd = i == 0, od = false;
        for (int j = 0; j < k.n_keys && i > 0; j++) {
            const uint8_t na = k.nul[j][i - 1], nb = k.nul[j][i];
            const uint64_t va = k.val[j][i - 1], vb = k.val[j][i];
            bool differ = na != nb || (!na && va != vb);
            if (j >= k.n_part && differ && !na && !nb && k.is_f64[j] && ((va | vb) << 1) == 0) differ = false;   // -0.0 == +0.0
            if (j < k.n_part) pd |= differ; else od |= differ;
        }
        part[i] = pd ? 1 : 0;
        peer[i] = (pd || od) ? 1 : 0;
    }
}

// ---- segmented scan ----
// MIN / MAX of a FLOAT / DOUBLE argument keep the earlier row of -0.0 and +0.0 in frame order, as the reference's strict
// ExprValue::compare does: the _F64 ops tie the two zeros; in a backward scan (_BWD) the left operand is the later row
enum ScanOp { SC_FIRST = 0, SC_SUM_I64, SC_SUM_F64, SC_MIN, SC_MAX, SC_MIN_F64, SC_MAX_F64, SC_MIN_F64_BWD, SC_MAX_F64_BWD };
enum ScanMode { SM_VALUE = 0, SM_INDEX = 1, SM_FLAG = 2 };
struct Acc { uint64_t v, c; uint32_t f; };
struct ScanIn {
    const uint64_t* v; const uint8_t* nul;   // SM_VALUE: value images (nullptr: every row counts, COUNT(*)) and null bytes
    const uint8_t* seg;                      // segment starts (forward order)
    const uint8_t* vflag;                    // SM_FLAG: the value is this byte (DENSE_RANK's peer starts)
    uint32_t n; int rev, mode, vclass;
};
constexpr int SC_THREADS = 256, SC_ITEMS = 8, SC_TILE = SC_THREADS * SC_ITEMS;

constexpr bool sc_is_min(int op) { return op == SC_MIN || op == SC_MIN_F64 || op == SC_MIN_F64_BWD; }
constexpr uint64_t IMG_NEG_ZERO = 0x7FFFFFFFFFFFFFFFull, IMG_POS_ZERO = 0x8000000000000000ull;   // ord_image of -0.0 / +0.0
// the key MIN / MAX compare: the order-preserving image, with -0.0 equal to +0.0 for FLOAT / DOUBLE
__device__ __forceinline__ uint64_t mm_key(uint64_t t, bool f64) { return f64 && t == IMG_NEG_ZERO ? IMG_POS_ZERO : t; }
// SUM's identity is -0.0, the one double x with -0.0 + x == x for every x: a frame of only -0.0 (and NULLs) sums to -0.0, as the
// reference's SUM (the first value, then the rest added) does
template <int OP> __device__ __forceinline__ uint64_t sc_ident() { return sc_is_min(OP) ? ~0ull : OP == SC_SUM_F64 ? 0x8000000000000000ull : 0ull; }
template <int OP> __device__ __forceinline__ Acc sc_identity() { Acc a; a.v = sc_ident<OP>(); a.c = 0; a.f = 0; return a; }
template <int OP> __device__ __forceinline__ Acc sc_comb(const Acc& a, const Acc& b) {
    if (b.f) return b;
    Acc r; r.f = a.f; r.c = a.c + b.c;
    if (OP == SC_FIRST) r.v = a.v;
    else if (OP == SC_SUM_I64) r.v = a.v + b.v;                                                     // two's-complement wrap
    else if (OP == SC_SUM_F64) r.v = __double_as_longlong(__longlong_as_double(a.v) + __longlong_as_double(b.v));
    else {                                                                                           // order-preserving images
        constexpr bool f64 = OP >= SC_MIN_F64, bwd = OP >= SC_MIN_F64_BWD;
        const uint64_t ka = mm_key(a.v, f64), kb = mm_key(b.v, f64);
        // b replaces a when strictly lower / higher; on a tie the backward scan takes b, the earlier row
        const bool take_b = sc_is_min(OP) ? (bwd ? kb <= ka : kb < ka) : (bwd ? kb >= ka : kb > ka);
        r.v = take_b ? b.v : a.v;
    }
    return r;
}
// order-preserving image of a value of class vclass (MIN / MAX compare these), and back
__device__ __forceinline__ uint64_t ord_image(uint64_t v, int vclass) {
    if (vclass == VC_F64) return (v >> 63) ? ~v : (v | 0x8000000000000000ull);
    if (vclass == VC_I64) return v ^ 0x8000000000000000ull;
    return v;
}
__device__ __forceinline__ uint64_t ord_value(uint64_t t, int vclass) {
    if (vclass == VC_F64) return (t >> 63) ? (t ^ 0x8000000000000000ull) : ~t;
    if (vclass == VC_I64) return t ^ 0x8000000000000000ull;
    return t;
}
template <int OP> __device__ __forceinline__ Acc sc_load(const ScanIn& in, uint32_t j) {
    if (j >= in.n) return sc_identity<OP>();
    const uint32_t p = in.rev ? in.n - 1 - j : j;
    Acc a;
    a.f = in.rev ? (j == 0 || in.seg[p + 1]) : in.seg[p];
    a.c = 1;
    if (in.mode == SM_INDEX) a.v = p;
    else if (in.mode == SM_FLAG) a.v = in.vflag[p];
    else if (!in.v) a.v = sc_ident<OP>();
    else if (in.nul[p]) { a.v = sc_ident<OP>(); a.c = 0; }
    else a.v = OP >= SC_MIN ? ord_image(in.v[p], in.vclass) : in.v[p];
    return a;
}
template <int OP> __device__ __forceinline__ Acc sc_shfl_up(const Acc& a, int d) {
    Acc r;
    r.v = __shfl_up_sync(0xFFFFFFFFu, a.v, d); r.c = __shfl_up_sync(0xFFFFFFFFu, a.c, d); r.f = __shfl_up_sync(0xFFFFFFFFu, a.f, d);
    return r;
}
template <int OP> __device__ __forceinline__ Acc sc_warp_incl(Acc x) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const Acc y = sc_shfl_up<OP>(x, d); if (lane >= d) x = sc_comb<OP>(y, x); }
    return x;
}
// exclusive prefix of each thread's aggregate within the CTA; `total` receives the CTA's aggregate
template <int OP> __device__ __forceinline__ Acc sc_block_excl(const Acc& t, Acc& total) {
    __shared__ Acc s_w[SC_THREADS / 32];
    __shared__ Acc s_total;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const Acc incl = sc_warp_incl<OP>(t);
    Acc excl = sc_shfl_up<OP>(incl, 1);
    if (lane == 0) excl = sc_identity<OP>();
    if (lane == 31) s_w[w] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
        Acc run = sc_identity<OP>();
        for (int k = 0; k < SC_THREADS / 32; k++) { const Acc x = s_w[k]; s_w[k] = run; run = sc_comb<OP>(run, x); }
        s_total = run;
    }
    __syncthreads();
    const Acc r = sc_comb<OP>(s_w[w], excl);
    total = s_total;
    __syncthreads();
    return r;
}
template <int OP> __global__ void __launch_bounds__(SC_THREADS) k_scan_reduce(ScanIn in, Acc* tile_agg) {
    const uint32_t j0 = blockIdx.x * SC_TILE + threadIdx.x * SC_ITEMS;
    Acc t = sc_identity<OP>();
#pragma unroll
    for (int k = 0; k < SC_ITEMS; k++) t = sc_comb<OP>(t, sc_load<OP>(in, j0 + k));
    Acc total;
    sc_block_excl<OP>(t, total);
    if (threadIdx.x == 0) tile_agg[blockIdx.x] = total;
}
// one CTA: exclusive prefix of the tile aggregates, SC_THREADS tiles per round (100M rows: 48k tiles, 191 rounds)
template <int OP> __global__ void __launch_bounds__(SC_THREADS) k_scan_tiles(const Acc* tile_agg, Acc* tile_carry, uint32_t ntiles) {
    __shared__ Acc s_carry;
    if (threadIdx.x == 0) s_carry = sc_identity<OP>();
    __syncthreads();
    for (uint32_t base = 0; base < ntiles; base += SC_THREADS) {
        const uint32_t i = base + threadIdx.x;
        const Acc x = i < ntiles ? tile_agg[i] : sc_identity<OP>();
        Acc total;
        const Acc excl = sc_block_excl<OP>(x, total);   // (ends with a barrier)
        const Acc carry = s_carry;
        if (i < ntiles) tile_carry[i] = sc_comb<OP>(carry, excl);
        __syncthreads();
        if (threadIdx.x == 0) s_carry = sc_comb<OP>(carry, total);
        __syncthreads();
    }
}
// inclusive scan value / count of every element, stored at its position in forward order
template <int OP> __global__ void __launch_bounds__(SC_THREADS) k_scan_down(ScanIn in, const Acc* tile_carry, uint64_t* out_v, uint64_t* out_c) {
    const uint32_t j0 = blockIdx.x * SC_TILE + threadIdx.x * SC_ITEMS;
    Acc el[SC_ITEMS];
    Acc t = sc_identity<OP>();
#pragma unroll
    for (int k = 0; k < SC_ITEMS; k++) { el[k] = sc_load<OP>(in, j0 + k); t = sc_comb<OP>(t, el[k]); }
    Acc total;
    const Acc excl = sc_block_excl<OP>(t, total);
    Acc run = sc_comb<OP>(tile_carry[blockIdx.x], excl);
#pragma unroll
    for (int k = 0; k < SC_ITEMS; k++) {
        const uint32_t j = j0 + k;
        if (j >= in.n) break;
        run = sc_comb<OP>(run, el[k]);
        const uint32_t p = in.rev ? in.n - 1 - j : j;
        out_v[p] = run.v;
        if (out_c) out_c[p] = run.c;
    }
}

// ---- one window function ----
struct FnArgs {
    int kind, method, has_order, arg_vclass, out_stype;
    int64_t n, param;
    const uint64_t *ps, *pl, *qs, *ql;   // partition start / last row, peer-group start / last row (sorted positions)
    const uint64_t* arg; const uint8_t* arg_nul;
    const uint64_t* def; const uint8_t* def_nul;
    const uint64_t *sv, *sc;             // scan value / count (WM_FWD, WM_BWD, WM_PEER); DENSE_RANK: count of peer starts in sv
    int has_frame, ftype, s_type, s_unb, e_type, e_unb;
    int64_t s_num, e_num;
    const uint32_t* perm;
    uint8_t* out_vals; uint8_t* out_null;
};

__device__ __forceinline__ void store_typed(uint8_t* vals, int stype, int64_t row, uint64_t v) {
    switch (stype) {
        case ST_I32: ((int32_t*)vals)[row] = (int32_t)(int64_t)v; break;
        case ST_U32: ((uint32_t*)vals)[row] = (uint32_t)v; break;
        case ST_F32: ((float*)vals)[row] = (float)__longlong_as_double(v); break;
        case ST_U8: vals[row] = v ? 1 : 0; break;
        default: ((uint64_t*)vals)[row] = v; break;
    }
}

__global__ void k_win_fn(FnArgs a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t ps = (int64_t)a.ps[i], pe = (int64_t)a.pl[i] + 1, size = pe - ps, r = i - ps;
        uint64_t v = 0; bool isnull = false;
        // the frame [fs, fe): RowFrameWindowProcessor / RangeFrameWindowProcessor::get_start_row / get_end_row, clamped to the partition
        int64_t fs = ps, fe = pe;
        if (a.has_frame) {
            if (!a.s_unb) {
                if (a.ftype == BK_FRAME_RANGE) fs = (int64_t)a.qs[i];
                else if (a.s_type == BK_BT_PRECEDING) fs = r >= a.s_num ? i - a.s_num : ps;
                else if (a.s_type == BK_BT_FOLLOWING) fs = r + a.s_num < size ? i + a.s_num : pe;
                else fs = i;
            }
            if (!a.e_unb) {
                if (a.ftype == BK_FRAME_RANGE) fe = (int64_t)a.ql[i] + 1;
                else if (a.e_type == BK_BT_PRECEDING) fe = r >= a.e_num ? i - a.e_num + 1 : ps;
                else if (a.e_type == BK_BT_FOLLOWING) fe = r + a.e_num < size ? i + a.e_num + 1 : pe;
                else fe = i + 1;
            }
        }
        const bool empty = fs >= fe;
        switch (a.kind) {
            case WF_ROW_NUMBER: v = (uint64_t)(r + 1); break;
            case WF_RANK: v = a.has_order ? (uint64_t)((int64_t)a.qs[i] - ps + 1) : 1; break;
            case WF_DENSE_RANK: v = a.has_order ? a.sv[i] : 1; break;
            case WF_PERCENT_RANK: {
                const double pr = (!a.has_order || size == 1) ? 0.0 : (double)((int64_t)a.qs[i] - ps) / (double)(size - 1);
                v = (uint64_t)__double_as_longlong(pr);
            } break;
            case WF_CUME_DIST: v = (uint64_t)__double_as_longlong(a.has_order ? (double)((int64_t)a.ql[i] + 1 - ps) / (double)size : 1.0); break;
            case WF_NTILE: {   // quotient / remainder buckets: the first `rem` buckets hold q + 1 rows
                const int64_t q = size / a.param, rem = size % a.param, big = rem * (q + 1);
                v = (uint64_t)(r < big ? r / (q + 1) + 1 : rem + (r - big) / q + 1);
            } break;
            case WF_LEAD: case WF_LAG: {   // (offsets up to INT64_MAX: compared with the distance to the partition's edge, never added)
                const bool inside = a.kind == WF_LEAD ? a.param < pe - i : a.param <= i - ps;
                if (inside) { const int64_t j = a.kind == WF_LEAD ? i + a.param : i - a.param; v = a.arg[j]; isnull = a.arg_nul[j]; }
                else if (a.def) { v = a.def[i]; isnull = a.def_nul[i]; }
                else isnull = true;
            } break;
            case WF_FIRST_VALUE: case WF_LAST_VALUE: case WF_NTH_VALUE: {
                // (NTH_VALUE: n is compared with the frame's width, so fs + n - 1 is only formed when it lies inside the frame)
                if (empty || (a.kind == WF_NTH_VALUE && a.param > fe - fs)) isnull = true;
                else {
                    const int64_t j = a.kind == WF_FIRST_VALUE ? fs : (a.kind == WF_LAST_VALUE ? fe - 1 : fs + a.param - 1);
                    v = a.arg[j]; isnull = a.arg_nul[j];
                }
            } break;
            default: {   // COUNT(*) COUNT SUM AVG MIN MAX over the frame
                uint64_t acc = 0, cnt = 0;
                if (!empty) {
                    if (a.method == WM_DIRECT) {
                        const bool is_min = a.kind == WF_MIN, is_max = a.kind == WF_MAX, f64 = a.arg_vclass == VC_F64;
                        acc = is_min ? ~0ull : 0ull;
                        double dacc = -0.0; bool dsum = false;   // (SUM's identity, as in the scans)
                        for (int64_t j = fs; j < fe; j++) {
                            if (a.kind == WF_COUNT_STAR) { cnt++; continue; }
                            if (a.arg_nul[j]) continue;
                            const uint64_t x = a.arg[j];
                            cnt++;
                            if (is_min || is_max) {   // the first value, then strictly lower / higher ones (the earlier of equal zeros stays)
                                const uint64_t t = ord_image(x, a.arg_vclass), kt = mm_key(t, f64), ka = mm_key(acc, f64);
                                if (cnt == 1 || (is_min ? kt < ka : kt > ka)) acc = t;
                            }
                            else if (a.kind == WF_AVG || (a.kind == WF_SUM && a.arg_vclass == VC_F64)) { dacc += __longlong_as_double(x); dsum = true; }
                            else acc += x;
                        }
                        if (dsum) acc = (uint64_t)__double_as_longlong(dacc);
                    } else {
                        const int64_t at = a.method == WM_BWD ? fs : fe - 1;
                        acc = a.sv[at]; cnt = a.sc[at];
                    }
                }
                if (a.kind == WF_COUNT_STAR || a.kind == WF_COUNT) v = cnt;
                else if (cnt == 0) isnull = true;
                else if (a.kind == WF_AVG) v = (uint64_t)__double_as_longlong((__longlong_as_double(acc) + 0.0) / (double)cnt);   // (the reference's AVG sum starts at +0.0)
                else if (a.kind == WF_MIN || a.kind == WF_MAX) v = ord_value(acc, a.arg_vclass);
                else v = acc;
            }
        }
        const int64_t row = (int64_t)a.perm[i];
        store_typed(a.out_vals, a.out_stype, row, isnull ? 0ull : v);
        a.out_null[row] = isnull ? 1 : 0;
    }
}

struct ScanBufs { Acc* agg = nullptr; Acc* carry = nullptr; uint32_t ntiles = 0; };

template <int OP> void launch_scan(const ScanIn& in, const ScanBufs& b, uint64_t* out_v, uint64_t* out_c, cudaStream_t st) {
    k_scan_reduce<OP><<<b.ntiles, SC_THREADS, 0, st>>>(in, b.agg);
    k_scan_tiles<OP><<<1, SC_THREADS, 0, st>>>(b.agg, b.carry, b.ntiles);
    k_scan_down<OP><<<b.ntiles, SC_THREADS, 0, st>>>(in, b.carry, out_v, out_c);
}
void run_scan(int op, const ScanIn& in, const ScanBufs& b, uint64_t* out_v, uint64_t* out_c, cudaStream_t st) {
    switch (op) {
        case SC_FIRST: launch_scan<SC_FIRST>(in, b, out_v, out_c, st); break;
        case SC_SUM_I64: launch_scan<SC_SUM_I64>(in, b, out_v, out_c, st); break;
        case SC_SUM_F64: launch_scan<SC_SUM_F64>(in, b, out_v, out_c, st); break;
        case SC_MIN: launch_scan<SC_MIN>(in, b, out_v, out_c, st); break;
        case SC_MAX: launch_scan<SC_MAX>(in, b, out_v, out_c, st); break;
        case SC_MIN_F64: launch_scan<SC_MIN_F64>(in, b, out_v, out_c, st); break;
        case SC_MAX_F64: launch_scan<SC_MAX_F64>(in, b, out_v, out_c, st); break;
        case SC_MIN_F64_BWD: launch_scan<SC_MIN_F64_BWD>(in, b, out_v, out_c, st); break;
        default: launch_scan<SC_MAX_F64_BWD>(in, b, out_v, out_c, st); break;
    }
}

}  // namespace

int window_finish(bkgpu_plan* p, const Compiled& c, SortState* rows, SortState* outer, bkgpu_stats* stats) {
    const cudaStream_t st = p->stream;
    const int sm = p->sm_count;
    DevScope ar(p);   // every device buffer of the call
    const RowStore& ret = sort_retained(rows);
    const int64_t n = ret.rows;
    if (n > RADIX_MAX_KEYS) return p->fail(BKGPU_EUNSUPPORTED, "a window fragment is limited to 2^30 - 1 rows per GPU");
    const int ncols = (int)ret.cols.size();
    int rc;
    // the retained rows as device columns: every bitmap packed from the null bytes
    std::vector<DevCol> cols(ret.cols.size());
    for (int k = 0; k < ncols; k++)
        if ((rc = store_pack(p, ret, (size_t)k, n, 8, nullptr, &cols[(size_t)k]))) return rc;
    uint32_t* perm = nullptr;
    if ((rc = ar.alloc(&perm, (size_t)n * 4))) return rc;
    if (n) k_iota<<<grid_for(n, sm, 8), 256, 0, st>>>(perm, n);
    // the output rows: the retained scan columns, then the window outputs (buffers of this call), in row space
    RowStore all = ret;
    for (const WinStage& w : c.win)
        for (const WinFn& f : w.fns) {
            RowStore::Col o; o.prim = f.out_prim;
            if ((rc = ar.alloc(&o.vals, (size_t)std::max<int64_t>(n, 1) * storage_bytes(prim_storage(f.out_prim)))) || (rc = ar.alloc(&o.nulls, (size_t)std::max<int64_t>(n, 1))))
                return rc;
            all.cols.push_back(o);
        }
    StageTimer timer;
    cudaEvent_t e0 = timer.a, e1 = timer.b;
    float win_ms = 0; int64_t win_bytes = 0, win_launches = 0;
    size_t fn_index = 0;
    const uint32_t ntiles = (uint32_t)((n + SC_TILE - 1) / SC_TILE);
    ScanBufs sb; sb.ntiles = ntiles;
    if ((rc = ar.alloc(&sb.agg, (size_t)std::max<uint32_t>(ntiles, 1) * sizeof(Acc))) || (rc = ar.alloc(&sb.carry, (size_t)std::max<uint32_t>(ntiles, 1) * sizeof(Acc))))
        return rc;
    for (const WinStage& w : c.win) {
        if (w.new_sort && n > 0) {   // stable radix sort of the current order by the stage's keys (each key: output 0 of its own program)
            std::vector<SortKey> keys; std::vector<const Program*> progs;
            for (const SortKey& k : w.sort_keys) { keys.push_back({0, k.prim, k.asc, k.null_first}); progs.push_back(&w.exprs[(size_t)k.out_reg]); }
            if ((rc = sort_stable_ids(rows, cols.data(), n, keys, progs, perm, stats))) return rc;
        }
        if (n == 0) { fn_index += w.fns.size(); continue; }
        cudaEventRecord(e0, st);
        // 1. expressions in sorted order
        std::vector<uint64_t*> ev(w.exprs.size()); std::vector<uint8_t*> en(w.exprs.size());
        EvalArgs ea; memset(&ea, 0, sizeof ea);
        for (int k = 0; k < ncols; k++) ea.cols[k] = cols[(size_t)k];
        ea.n_cols = ncols; ea.nrows = n;
        for (size_t e = 0; e < w.exprs.size(); e++) {
            if ((rc = ar.alloc(&ev[e], (size_t)n * 8)) || (rc = ar.alloc(&en[e], (size_t)n))) return rc;
            ea.prog = w.exprs[e];
            k_win_eval<<<grid_for(n, sm, 8), 256, 0, st>>>(ea, perm, ev[e], en[e]);
            win_launches++; win_bytes += n * (4 + 9);
        }
        // 2. partition / peer starts
        uint8_t *part = nullptr, *peer = nullptr;
        if ((rc = ar.alloc(&part, (size_t)n + 1)) || (rc = ar.alloc(&peer, (size_t)n + 1))) return rc;
        KeyCmp kc; memset(&kc, 0, sizeof kc);
        kc.n_part = w.n_part; kc.n_keys = (int)w.sort_keys.size();
        for (int k = 0; k < kc.n_keys; k++) {
            const SortKey& sk = w.sort_keys[(size_t)k];
            kc.val[k] = ev[(size_t)sk.out_reg]; kc.nul[k] = en[(size_t)sk.out_reg]; kc.is_f64[k] = host_prim_class(sk.prim) == VC_F64;
        }
        k_win_flags<<<grid_for(n, sm, 8), 256, 0, st>>>(kc, n, part, peer);
        win_launches++; win_bytes += n * (9 * 2 * kc.n_keys + 2);
        // 3. partition and peer-group bounds: the first index of the segment, forward and backward
        uint64_t *ps = nullptr, *pl = nullptr, *qs = nullptr, *ql = nullptr;
        if ((rc = ar.alloc(&ps, (size_t)n * 8)) || (rc = ar.alloc(&pl, (size_t)n * 8)) || (rc = ar.alloc(&qs, (size_t)n * 8)) || (rc = ar.alloc(&ql, (size_t)n * 8)))
            return rc;
        auto index_scan = [&](const uint8_t* seg, int rev, uint64_t* dst) {
            ScanIn in; memset(&in, 0, sizeof in);
            in.seg = seg; in.n = (uint32_t)n; in.rev = rev; in.mode = SM_INDEX;
            run_scan(SC_FIRST, in, sb, dst, nullptr, st);
            win_launches += 3; win_bytes += n * (2 + 8);
        };
        index_scan(part, 0, ps); index_scan(part, 1, pl); index_scan(peer, 0, qs); index_scan(peer, 1, ql);
        // 4. the functions
        uint64_t *sv = nullptr, *sc = nullptr;
        for (const WinFn& f : w.fns) {
            FnArgs fa; memset(&fa, 0, sizeof fa);
            fa.kind = f.kind; fa.method = f.method; fa.has_order = (int)w.sort_keys.size() > w.n_part; fa.n = n; fa.param = f.n;
            fa.ps = ps; fa.pl = pl; fa.qs = qs; fa.ql = ql;
            if (f.arg >= 0) { fa.arg = ev[(size_t)f.arg]; fa.arg_nul = en[(size_t)f.arg]; fa.arg_vclass = host_prim_class(f.arg_prim); }
            if (f.def >= 0) { fa.def = ev[(size_t)f.def]; fa.def_nul = en[(size_t)f.def]; }
            fa.has_frame = w.has_frame; fa.ftype = w.frame_type;
            fa.s_type = w.start.type; fa.s_unb = w.start.unbounded; fa.s_num = w.start.num;
            fa.e_type = w.end.type; fa.e_unb = w.end.unbounded; fa.e_num = w.end.num;
            const RowStore::Col& o = all.cols[(size_t)ncols + fn_index];
            fa.perm = perm; fa.out_vals = o.vals; fa.out_null = o.nulls; fa.out_stype = prim_storage(f.out_prim);
            const bool scanned = (f.kind <= WF_MAX && (f.method == WM_FWD || f.method == WM_BWD || f.method == WM_PEER)) || (f.kind == WF_DENSE_RANK && fa.has_order);
            if (scanned) {
                if (!sv && ((rc = ar.alloc(&sv, (size_t)n * 8)) || (rc = ar.alloc(&sc, (size_t)n * 8)))) return rc;
                ScanIn in; memset(&in, 0, sizeof in);
                in.n = (uint32_t)n; in.vclass = fa.arg_vclass;
                int op;
                if (f.kind == WF_DENSE_RANK) { in.mode = SM_FLAG; in.vflag = peer; in.seg = part; op = SC_SUM_I64; }
                else {
                    in.mode = SM_VALUE; in.v = fa.arg; in.nul = fa.arg_nul;
                    in.seg = f.method == WM_PEER ? peer : part; in.rev = f.method == WM_BWD;
                    op = f.kind == WF_MIN ? SC_MIN : f.kind == WF_MAX ? SC_MAX : (f.kind == WF_AVG || (f.kind == WF_SUM && fa.arg_vclass == VC_F64)) ? SC_SUM_F64 : SC_SUM_I64;
                    if (op == SC_MIN && fa.arg_vclass == VC_F64) op = in.rev ? SC_MIN_F64_BWD : SC_MIN_F64;
                    if (op == SC_MAX && fa.arg_vclass == VC_F64) op = in.rev ? SC_MAX_F64_BWD : SC_MAX_F64;
                }
                run_scan(op, in, sb, sv, sc, st);
                fa.sv = sv; fa.sc = sc;
                win_launches += 3; win_bytes += n * (2 * (9 + 1) + 16);
            }
            k_win_fn<<<grid_for(n, sm, 8), 256, 0, st>>>(fa);
            win_launches++; win_bytes += n * (4 * 8 + 4 + 9 + storage_bytes(fa.out_stype) + 1 + (scanned ? 16 : 0));
            fn_index++;
        }
        cudaEventRecord(e1, st);
        CK(p, cudaEventSynchronize(e1));
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1); win_ms += ms;
        for (size_t e = 0; e < ev.size(); e++) { ar.release(ev[e]); ar.release(en[e]); }
        for (void* b : {(void*)part, (void*)peer, (void*)ps, (void*)pl, (void*)qs, (void*)ql, (void*)sv, (void*)sc}) ar.release(b);
    }
    CK(p, cudaGetLastError());
    stats->main_kernel_ms += win_ms; stats->main_kernel_launches += 1; stats->main_kernel_bytes += win_bytes;
    stats->kernel_launches += win_launches;
    snprintf(stats->main_kernel_name, sizeof stats->main_kernel_name, "%s", "window_stage(k_win_fn)");
    std::vector<ColRef> desc;
    for (const OutCol& oc : c.out_cols) desc.push_back({oc.tuple_id, oc.slot_id, oc.prim});
    if (!outer) {
        int64_t keep = n;
        if (c.limit >= 0 && keep > c.limit) keep = c.limit;
        const int64_t skip = std::min<int64_t>(c.offset, keep);
        keep -= skip;
        return store_copy_out(p, all, desc, perm, keep, skip);
    }
    // the query's ORDER BY: the window rows in their order, as the post fragment's input, through its sort
    sort_reset(outer);
    bkgpu_stats scratch{};   // (the post fragment's kernels are not the request's main kernel)
    rc = sort_feed(outer, n, n, 8, &scratch, [&](RowStore& in) {
        int r = BKGPU_OK;
        for (size_t k = 0; k < in.cols.size() && !r; k++) r = store_gather(p, all.cols[k], perm, n, in.cols[k].vals, in.cols[k].nulls);
        return r;
    });
    if (!rc) rc = sort_finish(outer, nullptr, 1, &scratch, nullptr);
    stats->kernel_launches += scratch.kernel_launches;
    return rc;
}

}  // namespace bk

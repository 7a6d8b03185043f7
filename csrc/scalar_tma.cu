// scalar_tma.cu — the TMA-staged COUNT(*) WHERE `int32 column <cmp> constant` scan (config C1): the default for that shape
// (option "scalar_tma" = 0 pins the LDG kernel k_agg_scalar_direct<1,0> instead).
// north_star asks for "TMA-staged shared-memory tiles"; this is the kernel of the path where such a pipeline pays: one column, no
// tables in shared memory, pure streaming.
//
//   producer : one elected thread per CTA issues cp.async.bulk (1-D TMA, UBLKCP in SASS) of 16 KB column tiles into a 4-stage
//              shared-memory ring; each stage has a FULL mbarrier (armed with expect_tx, completed by the copy engine) and an EMPTY
//              mbarrier (one arrival per consumer thread)
//   consumers: all 256 threads wait on FULL (mbarrier.try_wait.parity), read the tile with conflict-free LDS.128, evaluate the
//              predicate ((x ^ m) <u t) != flip, arrive on EMPTY.  All six comparison operators fold into that one unsigned compare:
//              EQ / NE test (x ^ c) <u 1, LT / GE compare in the sign-biased domain (m = 2^31), LE / GT use c + 1 there
//              (c = INT32_MAX: a constant result)
// Replaces FilterNode::need_copy + AggFnCall::update(COUNT_STAR) for one batch (src/exec/filter_node.cpp:726-795,
// src/expr/agg_fn_call.cpp:496-555), like k_agg_scalar_direct<1, 0>.
#include "agg.h"
#include "dev_common.cuh"

namespace bk {

namespace {
constexpr int TMA_STAGES = 4;
constexpr int TMA_TILE_BYTES = 16384;
constexpr int TMA_THREADS = 256;

__device__ __forceinline__ uint32_t s_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

__global__ void __launch_bounds__(TMA_THREADS, 2) k_count_where_tma(const uint8_t* col, int64_t nrows, uint32_t m, uint32_t t, uint32_t flip,
                                                                     unsigned long long* rows_lane, unsigned long long* rows_passed) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t* bars = (uint64_t*)(smem + (size_t)TMA_STAGES * TMA_TILE_BYTES);   // [STAGES] full, [STAGES] empty
    const uint32_t full0 = s_addr(bars), empty0 = s_addr(bars + TMA_STAGES), tile0 = s_addr(smem);
    const int64_t ntiles = (nrows * 4) / TMA_TILE_BYTES;                         // whole tiles; the ragged rest is read directly
    if (threadIdx.x == 0) {
        for (int s = 0; s < TMA_STAGES; s++) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, TMA_THREADS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int64_t my_tiles = ntiles > blockIdx.x ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    uint32_t count = 0;
    // producer state (thread 0): tiles issued; consumer state: tiles consumed
    int64_t issued = 0;
    if (threadIdx.x == 0) {
        for (; issued < my_tiles && issued < TMA_STAGES; issued++) {
            const int s = (int)(issued % TMA_STAGES);
            mbar_expect_tx(full0 + 8 * s, TMA_TILE_BYTES);
            tma_load_1d(tile0 + s * TMA_TILE_BYTES, col + (size_t)(blockIdx.x + issued * gridDim.x) * TMA_TILE_BYTES, TMA_TILE_BYTES, full0 + 8 * s);
        }
    }
    for (int64_t k = 0; k < my_tiles; k++) {
        const int s = (int)(k % TMA_STAGES);
        const uint32_t parity = (uint32_t)((k / TMA_STAGES) & 1);
        mbar_wait(full0 + 8 * s, parity);
        const uint32_t base = tile0 + s * TMA_TILE_BYTES + threadIdx.x * 16;
#pragma unroll
        for (int i = 0; i < TMA_TILE_BYTES / (TMA_THREADS * 16); i++) {
            uint32_t x0, x1, x2, x3;
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0), "=r"(x1), "=r"(x2), "=r"(x3) : "r"(base + i * TMA_THREADS * 16));
            count += ((((x0 ^ m) < t) ? 1u : 0u) ^ flip) + ((((x1 ^ m) < t) ? 1u : 0u) ^ flip) + ((((x2 ^ m) < t) ? 1u : 0u) ^ flip) + ((((x3 ^ m) < t) ? 1u : 0u) ^ flip);
        }
        mbar_arrive(empty0 + 8 * s);                                             // this thread is done with the stage
        if (threadIdx.x == 0 && issued < my_tiles) {                             // refill the stage once every consumer has left it
            mbar_wait(empty0 + 8 * s, parity);
            mbar_expect_tx(full0 + 8 * s, TMA_TILE_BYTES);
            tma_load_1d(tile0 + s * TMA_TILE_BYTES, col + (size_t)(blockIdx.x + issued * gridDim.x) * TMA_TILE_BYTES, TMA_TILE_BYTES, full0 + 8 * s);
            issued++;
        }
    }
    // ragged rest (< one tile): plain loads by the first CTA
    if (blockIdx.x == 0) {
        const int64_t first = ntiles * (TMA_TILE_BYTES / 4);
        for (int64_t r = first + threadIdx.x; r < nrows; r += TMA_THREADS) {
            const uint32_t x = __ldg((const uint32_t*)col + r);
            count += (((x ^ m) < t) ? 1u : 0u) ^ flip;
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) count += __shfl_xor_sync(0xFFFFFFFFu, count, d);
    if ((threadIdx.x & 31) == 0 && count) { atomicAdd(rows_lane, (unsigned long long)count); atomicAdd(rows_passed, (unsigned long long)count); }
}
}  // namespace

// COUNT(*) WHERE int32 column <cmp> c over one batch (select_agg_launch has checked the shape)
cudaError_t launch_count_where_tma(const AggArgs& a, int sm_count, cudaStream_t s, cudaEvent_t start) {
    const DevCol& c = a.cols[0];
    const DirectTerm& tm = a.direct.term[0];
    const int32_t ci = (int32_t)(int64_t)tm.cbits;
    uint32_t m, t, flip;
    switch (tm.cmp) {   // ((x ^ m) <u t) != flip
        case BK_FT_EQ: m = (uint32_t)ci; t = 1; flip = 0; break;
        case BK_FT_NE: m = (uint32_t)ci; t = 1; flip = 1; break;
        case BK_FT_LT: m = 0x80000000u; t = (uint32_t)ci ^ 0x80000000u; flip = 0; break;
        case BK_FT_GE: m = 0x80000000u; t = (uint32_t)ci ^ 0x80000000u; flip = 1; break;
        case BK_FT_LE: m = 0x80000000u; t = ci == INT32_MAX ? 0u : ((uint32_t)(ci + 1) ^ 0x80000000u); flip = ci == INT32_MAX; break;
        default: m = 0x80000000u; t = ci == INT32_MAX ? 0u : ((uint32_t)(ci + 1) ^ 0x80000000u); flip = ci != INT32_MAX; break;
    }
    const size_t smem = (size_t)TMA_STAGES * TMA_TILE_BYTES + 2 * TMA_STAGES * 8;
    cudaError_t e = cudaFuncSetAttribute(k_count_where_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int64_t ntiles = (a.nrows * 4) / TMA_TILE_BYTES;
    int grid = 2 * sm_count;
    if (ntiles < grid) grid = (int)(ntiles > 0 ? ntiles : 1);
    if (start) cudaEventRecord(start, s);
    k_count_where_tma<<<grid, TMA_THREADS, smem, s>>>((const uint8_t*)c.values, a.nrows, m, t, flip, (unsigned long long*)a.gt.lanes, (unsigned long long*)a.rows_passed);
    return cudaGetLastError();
}

}  // namespace bk

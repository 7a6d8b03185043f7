// agg.h — the argument blocks of the filter+aggregate kernels and the launchers that cross translation units: the direct kernels
// (agg_direct*.cu), the TMA-staged COUNT(*) WHERE (scalar_tma.cu) and the join that returns rows (agg.cu, called by join.cu).
#pragma once
#include <cuda_runtime.h>
#include "dev_types.h"

namespace bk {

// hash join (K4): open-addressed multimap from the cast build key image to the build row
struct JoinArgs {
    const uint64_t* keys;    // [cap] key images
    const uint32_t* rows;    // [cap] build row, 0xFFFFFFFF = free slot
    uint32_t cap_mask;
    int32_t enabled;
    int32_t probe_col;       // index into cols of the probe key
    int32_t probe_prim, cast_prim;
    // LEFT / SEMI / ANTI_SEMI (the build side = the reference's outer / driver table is the preserved side, join_node.cpp:1200-1276,
    // joiner.cpp:633-685): `matched[build row]` is set to 1 by the probe; the TAIL launch (tail = 1) walks the n_build build rows and emits the
    // unmatched ones (0) NULL-extended (LEFT), the matched ones (1) (SEMI) or the unmatched ones (0) (ANTI_SEMI).  2 = removed by the build
    // side's own filter: never in the multimap, never emitted
    int32_t join_type;       // pb::JoinType: 1 LEFT, 3 INNER, 4 SEMI, 5 ANTI_SEMI, 6 FULL (RIGHT arrives as LEFT with the children swapped)
    int32_t tail;
    uint8_t* matched;
    int64_t n_build;
};

// FK -> PK join fused into the lean aggregate: the GROUP BY key is a build-side (dimension) attribute reached through
// the probe row's foreign key.  At build time the attribute is composed onto the key index (attr_of_key), so the probe
// is ONE random 4-byte read per fact row (served from L2: a 10M-key dimension is 40 MB); rows without a partner drop
// out (inner join), which the filter mask already expresses.
struct JoinProbe {
    int32_t mode;                // 0 = off, 1 = dense index, 2 = packed (key32 << 32 | attr32) open-addressed table
    int32_t key_signed;          // probe key column is a signed 32-bit type (canonical image sign-extends)
    const uint32_t* attr;        // mode 1: attribute by (key image ^ bias) - dense_min
    const uint32_t* present;     // mode 1: build row per key, 0xFFFFFFFF = no such key; nullptr = every key of the range exists
    uint64_t dense_min, dense_size, bias;
    const uint64_t* packed;      // mode 2
    uint32_t packed_mask;
};

struct AggArgs {
    DevCol cols[MAX_COLS];   // direct kernels: ordered [predicate][key][value] columns
    int32_t n_cols;
    int32_t smem_cap_log2;   // log2 slots of the per-CTA shared table (0 = no shared table)
    int64_t nrows;
    AggPlan plan;
    DirectPlan direct;
    Program prog;            // generic path only
    GroupTable gt;
    uint64_t* rows_passed;   // device counter: rows that survived the filter
    JoinArgs join;
    uint8_t smem_lane[MAX_LANES];  // global lane -> shared lane of this batch, 0xFF = not held in shared memory
    int32_t n_smem_lanes;
    uint32_t alias_mask;     // global lanes that receive the shared row count at flush time
    ValOps vops[4];          // direct kernels: per value column
    int32_t smem_keyw;       // key words per slot of the shared table (1 in sentinel mode, else plan.n_keyw)
    int32_t smem_paired;     // shared lanes are interleaved in 16-byte pairs {lane 2p, lane 2p+1} per slot (lean kernel: ATOMS.CAS.128)
    int32_t lean;            // batch qualifies for k_agg_group_lean (see agg_direct.cuh)
    int32_t smem_sentinel;   // shared table of one-word keys: the key word doubles as slot state (EMPTY_KEY = free)
    JoinProbe jp;            // lean kernel only: the key column holds the probe-side foreign key (see JoinProbe)
    int32_t lean_nulls;      // lean kernel: some predicate / value column of this batch carries a validity bitmap
    int32_t lean_mm;         // lean kernel: some value column feeds MIN / MAX lanes or more than one lane
    int32_t scalar_tma;      // 1 = try the TMA-staged scalar kernel (scalar_tma.cu)
    int32_t lean_fx;         // 1 = the lean kernel accumulates its double sums as fixed-point limbs with native 32-bit shared atomics (FX, agg_direct.cuh)
    uint32_t fx_ext_off;     // FX: byte offset (in the CTA's dynamic shared memory) of the low-extension limb arrays [value column][slot]
    // lean kernel: the last CTA to finish extracts the table's rows into this mapped host buffer (fused_extract, agg_kernels.cuh):
    // [32-byte counter block][values n_img x n][null bytes n_img x n], n = the groups in the table.  nullptr = no fused extraction
    uint8_t* fused_out;
    uint32_t fused_cap;      // rows the buffer holds: a table with more groups leaves only the counter block there (the host runs k_extract)
    // rb_build_agg: the pair buffer, one key per (row, AG_RB aggregate) with a non-NULL value: slot << 34 | rb_idx << 32 | low 32 bits of the
    // value.  *rb_ctr = keys appended (past rb_cap: keys were lost, the request fails with ETOOBIG).  nullptr without AG_RB
    uint64_t* rb_keys;
    unsigned long long* rb_ctr;
    uint64_t rb_cap;
};

// a row id that is no row: the NULL-extended side of an outer join's pair, a dimension without a partner in a star join's tuple
constexpr uint32_t JOIN_NO_ROW = 0xFFFFFFFFu;
enum AggKernel : int;   // agg_select.h: the kernel select_agg_launch chose for a batch
// scalar_tma.cu: TMA-staged COUNT(*) WHERE int32 <cmp> c (the batch has the kernel's shape)
cudaError_t launch_count_where_tma(const AggArgs& a, int sm_count, cudaStream_t s, cudaEvent_t start);
cudaError_t launch_direct_np0(const AggArgs& a, AggKernel k, int sm_count, size_t smem, cudaStream_t s, cudaEvent_t start);
cudaError_t launch_direct_np1(const AggArgs& a, AggKernel k, int sm_count, size_t smem, cudaStream_t s, cudaEvent_t start);
cudaError_t launch_direct_np2(const AggArgs& a, AggKernel k, int sm_count, size_t smem, cudaStream_t s, cudaEvent_t start);
// a JOIN that returns rows: (probe row, build row) pairs of the joined rows that pass the conditions, then one gather per output column
// (FULL, not the tail: k_join_pairs_full, which also emits the probe rows without a partner)
cudaError_t launch_join_pairs(const AggArgs& a, uint32_t* pairs, uint32_t cap, uint32_t* cursor, int sm_count, cudaStream_t s);

}  // namespace bk

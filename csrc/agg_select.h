// agg_select.h — which aggregate kernel runs a batch, and the per-batch fields of its AggArgs (agg_select.cpp).  Host only: it calls
// no CUDA function, so the whole choice can be checked on a machine without a GPU (tests/cpp/agg_select_check.cpp).
#pragma once
#include "agg.h"
#include "plan.h"

namespace bk {

// one value per launchable choice; the lean kernel's values are its instantiations (agg_direct.cuh: launch_direct)
enum AggKernel : int {
    INTERP,            // k_agg_interp: the bytecode interpreter, any plan
    SCALAR_DIRECT,     // k_agg_scalar_direct: no GROUP BY
    COUNT_WHERE_TMA,   // k_count_where_tma: COUNT(*) WHERE int32 <cmp> c (scalar_tma.cu)
    GROUP_DIRECT,      // k_agg_group_direct: the general direct GROUP BY kernel
    LEAN,              // k_agg_group_lean, plain CAS
    LEAN_NULLS,        // ... with validity bitmaps on predicate / value columns
    LEAN_MM,           // ... MIN / MAX or several lanes per column (with or without NULLs)
    LEAN_FX,           // ... double sums as fixed-point limbs
    LEAN_JOIN,         // ... with the fused FK -> PK probe
    LEAN_FX_JOIN,      // ... FX and the fused probe
};

// the name bkgpu_stats.main_kernel_name reports for a launch of `k`
const char* agg_kernel_name(AggKernel k);

// what the choice reads from the plan object: its options and the state learned from earlier launches
struct AggEnv {
    int force_generic = 0, no_lean = 0, no_lean_nulls = 0, no_lean_mm = 0;
    int lean_fx = 0, fx_off = 0;
    int scalar_tma = 0;
    int smem_cap_log2 = -1;       // -1 = chosen per batch from known_groups
    bool tail_launch = false;     // the outer-join tail: its probe-side columns are NULL on every row
    uint32_t known_groups = 0;    // groups seen by earlier launches of the plan
    bool multi_rank = false;      // the result is merged across ranks
    bool has_post = false;        // a post fragment (HAVING / SORT / LIMIT) runs above the aggregate
};

struct AggSelection {
    AggKernel kernel = INTERP;
    size_t smem = 0;              // dynamic shared memory of the INTERP and direct kernels (TMA sizes its own)
    bool fused_ok = false;        // the launch may extract its own result (fused_extract): the caller still has to get the buffer
};

// The kernel for one batch of `c` over `cols`, and every field of `a` except the device pointers gt, rows_passed, join and fused_out
// (`a` is cleared first).
// `vec_ok`: the columns allow the direct kernels' vector loads; `jp`: the fused FK -> PK probe.  Returns 0; +1 when `jp` is given and the
// batch does not fit the lean kernel; BKGPU_ENOMEM when the lean kernel's shared table does not fit.
int select_agg_launch(const Compiled& c, const DevCol* cols, int64_t nrows, bool vec_ok, const JoinProbe* jp, const AggEnv& env, AggArgs& a,
                      AggSelection& out);

// shared memory of the interpreter's table, of the direct kernels (table + queues) and of FX's extension limbs
size_t agg_smem_bytes(int smem_keyw, int n_smem_lanes, int cap_log2);
size_t direct_smem_bytes(int smem_keyw, int n_smem_lanes, int cap_log2, int na);
size_t fx_ext_bytes(int na, int cap_log2);

}  // namespace bk

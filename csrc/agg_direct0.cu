// agg_direct0.cu — instantiations of the direct filter+aggregate kernels with 0 predicate term(s)
// (one translation unit per term count so the library builds in parallel).
#include "agg_wp.cuh"

namespace bk {
cudaError_t launch_direct_np0(const AggArgs& a, int na, int sm_count, size_t smem, cudaStream_t s, bool grouped, cudaEvent_t start) {
    return launch_direct_np<0>(a, na, sm_count, smem, s, grouped, start);
}
}  // namespace bk

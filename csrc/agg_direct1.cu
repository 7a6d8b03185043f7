// agg_direct1.cu — instantiations of the direct filter+aggregate kernels with 1 predicate term(s)
// (one translation unit per term count so the library builds in parallel).
#include "agg_direct.cuh"

namespace bk {
cudaError_t launch_direct_np1(const AggArgs& a, AggKernel k, int sm_count, size_t smem, cudaStream_t s, cudaEvent_t start) {
    return launch_direct_np<1>(a, k, sm_count, smem, s, start);
}
}  // namespace bk

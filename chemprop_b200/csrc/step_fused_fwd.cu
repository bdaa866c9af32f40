// Instantiations of the fused depth-step kernel (csrc/step_fused_kernel.cuh); see csrc/step_fused.cu.
#include "step_fused_kernel.cuh"

namespace dmpnn {
namespace fused {
template cudaError_t dispatch_fwd<false>(int, bool, bool, bool, int, cudaStream_t, const CUtensorMap&, const Params&);
}  // namespace fused
}  // namespace dmpnn

// ATOM instantiations of the fused depth-step kernel (csrc/step_fused_kernel.cuh): the atom-granular step of
// AtomMessagePassing; see csrc/step_fused.cu (dmpnn_atom_step_fused_bf16).
#include "step_fused_kernel.cuh"

namespace dmpnn {
namespace fused {
template cudaError_t dispatch_bwd<false, true>(int, int, int, cudaStream_t, const CUtensorMap&, const Params&);
}  // namespace fused
}  // namespace dmpnn

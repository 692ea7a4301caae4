// Instantiations of the all-gather kernel for T = float (see launch_sra_inst for why they
// are not in sra_f32.cu).
#include "sra_kernels.cuh"

namespace cgx {
cudaError_t launch_ag_f32(const SraParams& p, cudaStream_t stream) { return launch_sra_t<float, kOpAllGather>(p, stream); }
}  // namespace cgx

// Instantiations of the all-gather kernel for T = __half (see launch_sra_inst for why they
// are not in sra_f16.cu).
#include "sra_kernels.cuh"

namespace cgx {
cudaError_t launch_ag_f16(const SraParams& p, cudaStream_t stream) { return launch_sra_t<__half, kOpAllGather>(p, stream); }
}  // namespace cgx

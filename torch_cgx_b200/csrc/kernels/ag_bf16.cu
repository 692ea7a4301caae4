// Instantiations of the all-gather kernel for T = __nv_bfloat16 (see launch_sra_inst for why they
// are not in sra_bf16.cu).
#include "sra_kernels.cuh"

namespace cgx {
cudaError_t launch_ag_bf16(const SraParams& p, cudaStream_t stream) { return launch_sra_t<__nv_bfloat16, kOpAllGather>(p, stream); }
}  // namespace cgx

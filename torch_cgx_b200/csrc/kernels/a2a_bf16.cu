// Instantiations of the all-to-all kernel for T = __nv_bfloat16 (see launch_sra_inst for why they are not in
// sra_bf16.cu).
#include "a2a_kernel.cuh"

namespace cgx {
cudaError_t launch_a2a_bf16(const A2aParams& p, cudaStream_t stream) { return launch_a2a_t<__nv_bfloat16>(p, stream); }
}  // namespace cgx

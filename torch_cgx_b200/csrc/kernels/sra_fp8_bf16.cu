// Instantiations of the FP8 allreduce kernels (sra_kernel / oneshot_kernel with an FP8 codec) for
// T = __nv_bfloat16 (see launch_sra_inst for why they are not in sra_bf16.cu).
#include "sra_kernels.cuh"

namespace cgx {
cudaError_t launch_sra_fp8_bf16(const SraParams& p, cudaStream_t stream) { return launch_sra_fp8_t<__nv_bfloat16>(p, stream); }
}  // namespace cgx

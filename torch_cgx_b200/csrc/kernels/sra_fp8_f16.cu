// Instantiations of the FP8 allreduce kernels (sra_kernel / oneshot_kernel with an FP8 codec) for
// T = __half (see launch_sra_inst for why they are not in sra_f16.cu).
#include "sra_kernels.cuh"

namespace cgx {
cudaError_t launch_sra_fp8_f16(const SraParams& p, cudaStream_t stream) { return launch_sra_fp8_t<__half>(p, stream); }
}  // namespace cgx

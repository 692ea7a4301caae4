// Instantiations of the FP8 allreduce kernels (sra_kernel / oneshot_kernel with an FP8 codec) for
// T = float (see launch_sra_inst for why they are not in sra_f32.cu).
#include "sra_kernels.cuh"

namespace cgx {
cudaError_t launch_sra_fp8_f32(const SraParams& p, cudaStream_t stream) { return launch_sra_fp8_t<float>(p, stream); }
}  // namespace cgx

// Instantiations of the reduce-scatter kernel for T = float (see launch_sra_inst for why they
// are not in sra_f32.cu).
#include "sra_kernels.cuh"

namespace cgx {
cudaError_t launch_rs_f32(const SraParams& p, cudaStream_t stream) { return launch_sra_t<float, kOpReduceScatter>(p, stream); }
}  // namespace cgx

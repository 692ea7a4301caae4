// Instantiations of the all-to-all kernel for T = float (see launch_sra_inst for why they are not in
// sra_f32.cu).
#include "a2a_kernel.cuh"

namespace cgx {
cudaError_t launch_a2a_f32(const A2aParams& p, cudaStream_t stream) { return launch_a2a_t<float>(p, stream); }
}  // namespace cgx

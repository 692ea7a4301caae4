// dtype dispatch of the fused kernels + occupancy query
#include "sra_kernels.cuh"

namespace cgx {

int sra_max_resident_ctas(int dtype) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int per_sm = 0;
  switch (dtype) {
    case kF32: per_sm = sra_resident_per_sm_f32(); break;
    case kF16: per_sm = sra_resident_per_sm_f16(); break;
    default: per_sm = sra_resident_per_sm_bf16(); break;
  }
  return sms * per_sm;
}

cudaError_t launch_sra_fused(const SraParams& p, cudaStream_t stream) {
  if (p.out != nullptr && p.gather) {
    switch (p.dtype) {
      case kF32: return launch_ag_f32(p, stream);
      case kF16: return launch_ag_f16(p, stream);
      case kBF16: return launch_ag_bf16(p, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  if (p.out != nullptr) {
    switch (p.dtype) {
      case kF32: return launch_rs_f32(p, stream);
      case kF16: return launch_rs_f16(p, stream);
      case kBF16: return launch_rs_bf16(p, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  if (p.codec != kMaxMin) {
    switch (p.dtype) {
      case kF32: return launch_sra_fp8_f32(p, stream);
      case kF16: return launch_sra_fp8_f16(p, stream);
      case kBF16: return launch_sra_fp8_bf16(p, stream);
      default: return cudaErrorInvalidValue;
    }
  }
  switch (p.dtype) {
    case kF32: return launch_sra_f32(p, stream);
    case kF16: return launch_sra_f16(p, stream);
    case kBF16: return launch_sra_bf16(p, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace cgx

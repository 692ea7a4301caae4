// The weighted top-k combine of slot rows that are already in memory: the composed path of the
// combine (process group over NCCL, rows the fused kernel cannot route, world 1 without a heap).
// One warp per (token, segment of kSegElems columns), the arithmetic of combine_segment, so the
// result equals the fused all-to-all's combine bit for bit.
#include "combine.cuh"
#include "launch.h"

namespace cgx {
using namespace dev;

namespace {
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kSegElems = 512;

template <typename T>
__global__ void __launch_bounds__(kThreads) combine_rows_kernel(const T* __restrict__ slots,
                                                                const float* __restrict__ gate, T* __restrict__ out,
                                                                uint64_t T_, uint32_t k, uint32_t H) {
  const uint32_t segs = (H + kSegElems - 1u) / kSegElems;
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t w = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); w < T_ * segs; w += nwarps) {
    const uint64_t t = w / segs;
    const uint32_t col = (uint32_t)(w - t * segs) * kSegElems;
    combine_segment<T>(slots + t * k * H + col, H, gate + t * k, k, out + t * H + col, min(kSegElems, H - col));
  }
}

template <typename T>
cudaError_t combine_rows_t(const void* slots, const float* gate, void* out, uint64_t T_, uint32_t k, uint32_t H,
                           cudaStream_t stream) {
  const uint64_t warps = T_ * ((H + kSegElems - 1u) / kSegElems);
  const int grid = (int)std::min<uint64_t>((warps + kWarps - 1) / kWarps, 1u << 16);
  combine_rows_kernel<T><<<grid, kThreads, 0, stream>>>((const T*)slots, gate, (T*)out, T_, k, H);
  return cudaGetLastError();
}
}  // namespace

cudaError_t launch_combine_rows(const void* slots, const float* gate, void* out, int dtype, uint64_t T, uint32_t k,
                                uint32_t H, cudaStream_t stream) {
  if (T == 0 || H == 0) return cudaSuccess;
  if (k < 1 || k > 32) return cudaErrorInvalidValue;
  switch (dtype) {
    case kF32: return combine_rows_t<float>(slots, gate, out, T, k, H, stream);
    case kF16: return combine_rows_t<__half>(slots, gate, out, T, k, H, stream);
    case kBF16: return combine_rows_t<__nv_bfloat16>(slots, gate, out, T, k, H, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace cgx

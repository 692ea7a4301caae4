// The weighted top-k combine of slot rows that are already in memory: the composed path of the
// combine (process group over NCCL, rows the fused kernel cannot route, world 1 without a heap).
// One warp per (token, segment of kSegElems columns), the arithmetic of combine_segment, so the
// result equals the fused all-to-all's combine bit for bit.
// Next to it, for the combine's backward (DESIGN §2.13e): the gate gradient in one pass over the
// slots, and the in-place scale of the composed path's scaled send.
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

// One warp per token t reads grad_out[t] once and the k <= KMAX slot rows t * k + c, and writes
// grad_gate[t, c] for every c. Lane l owns the V-element groups l, l + 32, ... of the row (V = 16 B
// of T) and runs acc_c = fma(go_h, x_h, acc_c) over its elements in increasing h, whatever the
// alignment: 16-byte loads where grad_out, the slots and the row length are 16-byte aligned, else
// the same elements one at a time. The butterfly acc_c += shfl_xor(acc_c, m), m = 16 .. 1, then
// leaves the sum in every lane, and lane c stores it. The accumulators are a KMAX array indexed by
// compile-time c only, so they stay in registers.
template <typename T, int KMAX>
__global__ void __launch_bounds__(kThreads) combine_gate_grad_kernel(const T* __restrict__ grad_out,
                                                                     const T* __restrict__ slots,
                                                                     float* __restrict__ grad_gate, uint64_t T_,
                                                                     uint32_t k, uint32_t H) {
  constexpr uint32_t V = (uint32_t)DT<T>::kVec;
  const uint32_t lane = lane_id(), groups = (H + V - 1u) / V;
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t t = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); t < T_; t += nwarps) {
    const T* go = grad_out + t * H;
    const T* x = slots + t * k * H;
    const bool vec = ((reinterpret_cast<uintptr_t>(go) | reinterpret_cast<uintptr_t>(x) | (uintptr_t)(H * sizeof(T))) &
                      15u) == 0;
    float acc[KMAX];
#pragma unroll
    for (int c = 0; c < KMAX; ++c) acc[c] = 0.f;
    for (uint32_t v = lane; v < groups; v += 32) {
      const uint32_t h0 = v * V;
      if (vec && h0 + V <= H) {
        float g[V];
        unpack16<T>(__ldcg(reinterpret_cast<const uint4*>(go + h0)), g);
#pragma unroll
        for (int c = 0; c < KMAX; ++c) {
          if ((uint32_t)c < k) {
            float xv[V];
            unpack16<T>(__ldcg(reinterpret_cast<const uint4*>(x + (uint64_t)c * H + h0)), xv);
#pragma unroll
            for (uint32_t i = 0; i < V; ++i) acc[c] = __fmaf_rn(g[i], xv[i], acc[c]);
          }
        }
      } else {
        const uint32_t m = min(V, H - h0);
        for (uint32_t i = 0; i < m; ++i) {
          const float g = ld_cg_float(go + h0 + i);
#pragma unroll
          for (int c = 0; c < KMAX; ++c)
            if ((uint32_t)c < k) acc[c] = __fmaf_rn(g, ld_cg_float(x + (uint64_t)c * H + h0 + i), acc[c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < KMAX; ++c) {
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) acc[c] = __fadd_rn(acc[c], __shfl_xor_sync(kAll, acc[c], m));
      if ((uint32_t)c < k && lane == (uint32_t)c) grad_gate[t * k + c] = acc[c];
    }
  }
}

template <typename T, int KMAX>
cudaError_t combine_gate_grad_k(const void* grad_out, const void* slots, float* grad_gate, uint64_t T_, uint32_t k,
                                uint32_t H, cudaStream_t stream) {
  const int grid = (int)std::min<uint64_t>((T_ + kWarps - 1) / kWarps, 1u << 16);
  combine_gate_grad_kernel<T, KMAX><<<grid, kThreads, 0, stream>>>((const T*)grad_out, (const T*)slots, grad_gate, T_,
                                                                   k, H);
  return cudaGetLastError();
}
template <typename T>
cudaError_t combine_gate_grad_t(const void* grad_out, const void* slots, float* grad_gate, uint64_t T_, uint32_t k,
                                uint32_t H, cudaStream_t stream) {
  if (k <= 1) return combine_gate_grad_k<T, 1>(grad_out, slots, grad_gate, T_, k, H, stream);
  if (k <= 2) return combine_gate_grad_k<T, 2>(grad_out, slots, grad_gate, T_, k, H, stream);
  if (k <= 4) return combine_gate_grad_k<T, 4>(grad_out, slots, grad_gate, T_, k, H, stream);
  if (k <= 8) return combine_gate_grad_k<T, 8>(grad_out, slots, grad_gate, T_, k, H, stream);
  if (k <= 16) return combine_gate_grad_k<T, 16>(grad_out, slots, grad_gate, T_, k, H, stream);
  return combine_gate_grad_k<T, 32>(grad_out, slots, grad_gate, T_, k, H, stream);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) scale_rows_kernel(T* __restrict__ rows, const float* __restrict__ scale,
                                                              uint64_t n, uint64_t H) {
  const uint64_t nthr = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += nthr)
    rows[i] = scale_round_to<T>(DT<T>::to_float(rows[i]), scale[i / H]);
}
template <typename T>
cudaError_t scale_rows_t(void* rows, const float* scale, uint64_t R, uint64_t H, cudaStream_t stream) {
  const uint64_t n = R * H;
  const int grid = (int)std::min<uint64_t>((n + kThreads - 1) / kThreads, 1u << 16);
  scale_rows_kernel<T><<<grid, kThreads, 0, stream>>>((T*)rows, scale, n, H);
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

cudaError_t launch_combine_gate_grad(const void* grad_out, const void* slots, float* grad_gate, int dtype, uint64_t T,
                                     uint32_t k, uint32_t H, cudaStream_t stream) {
  if (T == 0) return cudaSuccess;
  if (k < 1 || k > 32) return cudaErrorInvalidValue;
  switch (dtype) {
    case kF32: return combine_gate_grad_t<float>(grad_out, slots, grad_gate, T, k, H, stream);
    case kF16: return combine_gate_grad_t<__half>(grad_out, slots, grad_gate, T, k, H, stream);
    case kBF16: return combine_gate_grad_t<__nv_bfloat16>(grad_out, slots, grad_gate, T, k, H, stream);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_scale_rows(void* rows, const float* scale, int dtype, uint64_t R, uint64_t H, cudaStream_t stream) {
  if (R == 0 || H == 0) return cudaSuccess;
  switch (dtype) {
    case kF32: return scale_rows_t<float>(rows, scale, R, H, stream);
    case kF16: return scale_rows_t<__half>(rows, scale, R, H, stream);
    case kBF16: return scale_rows_t<__nv_bfloat16>(rows, scale, R, H, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace cgx

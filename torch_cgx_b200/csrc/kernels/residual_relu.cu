// Residual join of the ResNet blocks, y = relu(a + b), and its backward g = (y <= 0) ? 0 : ga + gb.
//
// Bit-identical to the eager composition it replaces:
//   forward   at::add (alpha 1: T(float(a) + float(b)), round to nearest even), then relu_ =
//             clamp_min(v, 0), which keeps a NaN as it is and turns -0 into +0;
//   backward  the autograd engine's accumulation of the two incoming gradients (at::add again), then
//             threshold_backward(grad, y, 0) = (y <= 0) ? 0 : grad, so a NaN y passes its gradient.
// Both are "keep v unless v <= 0, else +0" on the T value: relu(v) = (v <= 0) ? +0 : v.
// The extension is built with --fmad=false and the sum is an explicit __fadd_rn.
//
// All operands are dense with identical sizes and strides (checked by the binding), so the kernels
// walk the storage linearly: 16-byte vectors when every pointer is 16-byte aligned, otherwise one
// element per thread in a grid-stride loop.
#include "device_utils.cuh"
#include "launch.h"

namespace cgx {
using namespace dev;

namespace {
constexpr int kThreads = 256;
constexpr int kUnroll = 2;  // 16-byte vectors per operand and thread: 32 B of each input in flight

template <typename T>
__device__ __forceinline__ T relu_sum(T a, T b) {
  const float s = __fadd_rn(DT<T>::to_float(a), DT<T>::to_float(b));
  const T t = DT<T>::from_float(s);
  return DT<T>::to_float(t) <= 0.0f ? DT<T>::from_float(0.0f) : t;
}

template <typename T, bool HAS_GB>
__device__ __forceinline__ T relu_grad(T y, T ga, T gb) {
  if (DT<T>::to_float(y) <= 0.0f) return DT<T>::from_float(0.0f);
  if (!HAS_GB) return ga;
  return DT<T>::from_float(__fadd_rn(DT<T>::to_float(ga), DT<T>::to_float(gb)));
}

template <typename T>
union Vec16 {
  uint4 u;
  T e[DT<T>::kVec];
};

// ---- 16-byte path: every pointer 16-byte aligned; the n % kVec tail runs on the first threads
template <typename T>
__global__ void __launch_bounds__(kThreads)
residual_relu_fwd_vec(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ y, uint64_t n) {
  constexpr int V = DT<T>::kVec;
  const uint64_t nv = n / V;
  const uint4* a4 = reinterpret_cast<const uint4*>(a);
  const uint4* b4 = reinterpret_cast<const uint4*>(b);
  uint4* y4 = reinterpret_cast<uint4*>(y);
  const uint64_t step = (uint64_t)gridDim.x * kThreads * kUnroll;
  for (uint64_t base = (uint64_t)blockIdx.x * kThreads * kUnroll + threadIdx.x; base < nv; base += step) {
    Vec16<T> va[kUnroll], vb[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint64_t i = base + (uint64_t)u * kThreads;
      if (i < nv) {
        va[u].u = __ldg(a4 + i);
        vb[u].u = __ldg(b4 + i);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint64_t i = base + (uint64_t)u * kThreads;
      if (i < nv) {
        Vec16<T> vy;
#pragma unroll
        for (int j = 0; j < V; ++j) vy.e[j] = relu_sum<T>(va[u].e[j], vb[u].e[j]);
        y4[i] = vy.u;
      }
    }
  }
  const uint64_t t = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  if (t < n - nv * V) {
    const uint64_t i = nv * V + t;
    y[i] = relu_sum<T>(a[i], b[i]);
  }
}

template <typename T, bool HAS_GB>
__global__ void __launch_bounds__(kThreads)
residual_relu_bwd_vec(const T* __restrict__ y, const T* __restrict__ ga, const T* __restrict__ gb,
                      T* __restrict__ g, uint64_t n) {
  constexpr int V = DT<T>::kVec;
  const uint64_t nv = n / V;
  const uint4* y4 = reinterpret_cast<const uint4*>(y);
  const uint4* ga4 = reinterpret_cast<const uint4*>(ga);
  const uint4* gb4 = reinterpret_cast<const uint4*>(gb);
  uint4* g4 = reinterpret_cast<uint4*>(g);
  const uint64_t step = (uint64_t)gridDim.x * kThreads * kUnroll;
  for (uint64_t base = (uint64_t)blockIdx.x * kThreads * kUnroll + threadIdx.x; base < nv; base += step) {
    Vec16<T> vy[kUnroll], va[kUnroll], vb[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint64_t i = base + (uint64_t)u * kThreads;
      if (i < nv) {
        vy[u].u = __ldg(y4 + i);
        va[u].u = __ldg(ga4 + i);
        if (HAS_GB) vb[u].u = __ldg(gb4 + i);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint64_t i = base + (uint64_t)u * kThreads;
      if (i < nv) {
        Vec16<T> vg;
#pragma unroll
        for (int j = 0; j < V; ++j)
          vg.e[j] = relu_grad<T, HAS_GB>(vy[u].e[j], va[u].e[j], HAS_GB ? vb[u].e[j] : va[u].e[j]);
        g4[i] = vg.u;
      }
    }
  }
  const uint64_t t = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
  if (t < n - nv * V) {
    const uint64_t i = nv * V + t;
    g[i] = relu_grad<T, HAS_GB>(y[i], ga[i], HAS_GB ? gb[i] : ga[i]);
  }
}

// ---- scalar path: any element alignment
template <typename T>
__global__ void __launch_bounds__(kThreads)
residual_relu_fwd_scalar(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ y, uint64_t n) {
  const uint64_t stride = (uint64_t)gridDim.x * kThreads;
  for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) y[i] = relu_sum<T>(a[i], b[i]);
}

template <typename T, bool HAS_GB>
__global__ void __launch_bounds__(kThreads)
residual_relu_bwd_scalar(const T* __restrict__ y, const T* __restrict__ ga, const T* __restrict__ gb,
                         T* __restrict__ g, uint64_t n) {
  const uint64_t stride = (uint64_t)gridDim.x * kThreads;
  for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += stride)
    g[i] = relu_grad<T, HAS_GB>(y[i], ga[i], HAS_GB ? gb[i] : ga[i]);
}

bool aligned16(const void* p) { return p == nullptr || ((uintptr_t)p & 15u) == 0; }

// one vector (or tail element) per thread and unroll step; capped, the kernels loop beyond that
int vec_grid(uint64_t n, int vec) {
  const uint64_t per_block = (uint64_t)kThreads * kUnroll;
  uint64_t want = (n / vec + per_block - 1) / per_block;
  const uint64_t tail_blocks = ((uint64_t)(n % vec) + kThreads - 1) / kThreads;
  if (want < tail_blocks) want = tail_blocks;
  return (int)(want < 1 ? 1 : (want > (1u << 20) ? (1u << 20) : want));
}
int scalar_grid(uint64_t n) {
  const uint64_t want = (n + kThreads - 1) / kThreads;
  return (int)(want < 1 ? 1 : (want > 8192 ? 8192 : want));
}

template <typename T>
cudaError_t forward_t(const T* a, const T* b, T* y, uint64_t n, cudaStream_t stream) {
  if (aligned16(a) && aligned16(b) && aligned16(y))
    residual_relu_fwd_vec<T><<<vec_grid(n, DT<T>::kVec), kThreads, 0, stream>>>(a, b, y, n);
  else
    residual_relu_fwd_scalar<T><<<scalar_grid(n), kThreads, 0, stream>>>(a, b, y, n);
  return cudaGetLastError();
}

template <typename T>
cudaError_t backward_t(const T* y, const T* ga, const T* gb, T* g, uint64_t n, cudaStream_t stream) {
  const bool vec = aligned16(y) && aligned16(ga) && aligned16(gb) && aligned16(g);
  if (vec && gb)
    residual_relu_bwd_vec<T, true><<<vec_grid(n, DT<T>::kVec), kThreads, 0, stream>>>(y, ga, gb, g, n);
  else if (vec)
    residual_relu_bwd_vec<T, false><<<vec_grid(n, DT<T>::kVec), kThreads, 0, stream>>>(y, ga, gb, g, n);
  else if (gb)
    residual_relu_bwd_scalar<T, true><<<scalar_grid(n), kThreads, 0, stream>>>(y, ga, gb, g, n);
  else
    residual_relu_bwd_scalar<T, false><<<scalar_grid(n), kThreads, 0, stream>>>(y, ga, gb, g, n);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_residual_relu_forward(const void* a, const void* b, void* y, int dtype, uint64_t n,
                                         cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  switch (dtype) {
    case kF32: return forward_t<float>((const float*)a, (const float*)b, (float*)y, n, stream);
    case kF16: return forward_t<__half>((const __half*)a, (const __half*)b, (__half*)y, n, stream);
    case kBF16:
      return forward_t<__nv_bfloat16>((const __nv_bfloat16*)a, (const __nv_bfloat16*)b, (__nv_bfloat16*)y, n, stream);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_residual_relu_backward(const void* y, const void* ga, const void* gb, void* g, int dtype,
                                          uint64_t n, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  switch (dtype) {
    case kF32: return backward_t<float>((const float*)y, (const float*)ga, (const float*)gb, (float*)g, n, stream);
    case kF16: return backward_t<__half>((const __half*)y, (const __half*)ga, (const __half*)gb, (__half*)g, n, stream);
    case kBF16:
      return backward_t<__nv_bfloat16>((const __nv_bfloat16*)y, (const __nv_bfloat16*)ga, (const __nv_bfloat16*)gb,
                                       (__nv_bfloat16*)g, n, stream);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace cgx

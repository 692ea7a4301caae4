// Standalone item kernels: the same warp-item device primitives as the fused kernel, one launch
// over MANY items (one warp per item, grid-stride), used by the generic reducers (SRA / Ring over
// NCCL send/recv = the cross-node path and the "reference-structure" baseline), by the Python ops
// and by the tests. Covers K1-K5/K7 of SURVEY.md §2.3
// (/root/reference/src/common/compression/cuda_compression_operations.cu:58-65, :98-153,
// :287-371, :474-544, :583-598, :784-798).
#include "item_ops.cuh"
#include "launch.h"

namespace cgx {
using namespace dev;

namespace {
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ uint32_t global_warp() { return blockIdx.x * kWarps + (threadIdx.x >> 5); }
__device__ __forceinline__ uint32_t total_warps() { return gridDim.x * kWarps; }

// Each warp walks items first+w, first+w+stride, ...; the descriptor of the NEXT item is loaded
// before the current one is processed so that its latency hides behind the work.
#define CGX_ITEM_LOOP(it)                                                       \
  const uint32_t stride_ = total_warps();                                       \
  uint32_t i_ = global_warp();                                                  \
  WarpItem it, next_;                                                           \
  if (i_ < count) it = items[first + i_];                                       \
  for (; i_ < count; i_ += stride_, it = next_)                                 \
    if (next_ = (i_ + stride_ < count) ? items[first + i_ + stride_] : it, true)

// wire = quantize(src * prescale); TS = T (tensor) or float (fp32 scratch indexed from base_elem);
// out != nullptr: also write the self-decoded values (T, indexed from the tensor base)
template <typename TS, typename T, int KB, int GPL>
__global__ void __launch_bounds__(kThreads, 3)
quantize_items_kernel(const TS* __restrict__ src, uint32_t base_elem, const WarpItem* __restrict__ items,
                      uint32_t first, uint32_t count, uint8_t* wire, float prescale, const RngKey rng,
                      T* __restrict__ out) {
  const OneDst ds{wire};
  const SrcSet no_src{nullptr, 0u, 0, -1};
  CGX_ITEM_LOOP(it) {
    const uint32_t kind = item_kind(it);
    const TS* s = src + (it.elem_off - base_elem);
    T* o = out ? out + it.elem_off : nullptr;
    if (i_ + stride_ < count) slice_prefetch_l2<TS, GPL>(src + (next_.elem_off - base_elem));
    if (kind == kItemFull) {
      const bool al = group_aligned<TS>(s) && (o == nullptr || group_aligned<T>(o));
      if (al) {
        float x[GPL][8];
        slice_load_vec<TS, GPL>(s, x);
        if (o)
          full_send_x<T, KB, GPL, true, true>(x, it, prescale, rng, ds, o);
        else
          full_send_x<T, KB, GPL, false, true>(x, it, prescale, rng, ds, o);
      } else if (o) {
        full_send_unaligned<TS, T, KB, GPL, true>(s, it, prescale, rng, ds, o);
      } else {
        full_send_unaligned<TS, T, KB, GPL, false>(s, it, prescale, rng, ds, o);
      }
    } else if (kind == kItemBucket) {
      bucket_quantize<TS, T>(s, it, prescale, rng, no_src, ds, o);
    } else {
      // raw items travel as T: wire <- T(src * prescale) [, out <- the same]
      const uint32_t n = item_n(it);
      T* w = reinterpret_cast<T*>(wire + it.meta_off);
      for (uint32_t e = lane_id(); e < n; e += 32) {
        const T t = DT<T>::from_float(__fmul_rn(DT<TS>::to_float(s[e]), prescale));
        w[e] = t;
        if (o) o[e] = t;
      }
    }
  }
}

template <typename T, int KB, int GPL>
__global__ void __launch_bounds__(kThreads, 3)
dequantize_items_kernel(const uint8_t* __restrict__ wire, const WarpItem* __restrict__ items, uint32_t first,
                        uint32_t count, T* __restrict__ dst) {
  const SrcSet ss{wire, 0u, 1, -1};
  CGX_ITEM_LOOP(it) {
    const uint32_t kind = item_kind(it);
    T* o = dst + it.elem_off;
    if (i_ + stride_ < count && lane_id() < 4u)  // the next item's packed words (<= 1 KB) and meta
      asm volatile("prefetch.global.L2 [%0];" ::"l"(wire + (lane_id() == 3u ? next_.meta_off : next_.pay_off + lane_id() * 256u)));
    if (kind == kItemFull) {
      if (group_aligned<T>(o)) {
        SliceWords<GPL> w;
        slice_fetch<KB, GPL>(wire, it.meta_off, it.pay_off, item_lpb_log2(it), KB ? KB : item_bits(it), w);
        full_recv_w<T, KB, GPL, true>(w, it, o);
      } else {
        full_recv_unaligned<T, KB, GPL>(ss, it, o);
      }
    } else if (kind == kItemBucket) {
      bucket_recv<T>(ss, it, o);
    } else {
      const uint32_t n = item_n(it);
      const T* w = reinterpret_cast<const T*>(wire + it.meta_off);
      for (uint32_t e = lane_id(); e < n; e += 32) o[e] = w[e];
    }
  }
}

// acc (fp32 scratch) = float(init_src) * prescale   (init_src != nullptr)
// acc += decode(wire)                                (wire != nullptr)
template <typename T, int KB, int GPL>
__global__ void __launch_bounds__(kThreads, 3)
accumulate_items_kernel(const uint8_t* __restrict__ wire, const WarpItem* __restrict__ items, uint32_t first,
                        uint32_t count, float* __restrict__ acc, uint32_t base_elem, const T* __restrict__ init_src,
                        float prescale) {
  CGX_ITEM_LOOP(it) {
    const uint32_t kind = item_kind(it);
    float* a = acc + (it.elem_off - base_elem);
    if (kind == kItemFull) {
      const int bits = KB ? KB : item_bits(it);
      const uint32_t lg = item_lpb_log2(it);
      float x[GPL][8];
      if (init_src) {
        const T* s = init_src + it.elem_off;
        if (group_aligned<T>(s))
          slice_load_vec<T, GPL>(s, x);
        else
          slice_load_scalar<T, GPL>(s, x);
        slice_scale<GPL>(x, prescale);
      } else if (group_aligned<float>(a)) {
        slice_load_vec<float, GPL>(a, x);
      } else {
        slice_load_scalar<float, GPL>(a, x);
      }
      if (wire) {
        SliceWords<GPL> w;
        slice_fetch<KB, GPL>(wire, it.meta_off, it.pay_off, lg, bits, w);
        slice_decode<KB, GPL, true>(w, bits, x);
      }
      if (group_aligned<float>(a))
        slice_store<float, GPL, true>(a, x);
      else
        slice_store<float, GPL, false>(a, x);
    } else if (kind == kItemBucket) {
      const uint32_t n = item_n(it);
      const int bits = item_bits(it);
      const uint32_t ng = div_up(n, 8u);
      for (uint32_t g = lane_id(); g < ng; g += 32) {
        const int nv = (int)min(8u, n - g * 8u);
        float x[8];
        if (init_src) {
          load8_scalar<T>(init_src + it.elem_off + g * 8u, nv, x);
#pragma unroll
          for (int j = 0; j < 8; ++j) x[j] = __fmul_rn(x[j], prescale);
        } else {
          load8_scalar<float>(a + g * 8u, nv, x);
        }
        if (wire) bucket_add_sources(SrcSet{wire, 0u, 1, -1}, it, g, bits, x);
        store8_scalar<float>(a + g * 8u, nv, x);
      }
    } else {
      const uint32_t n = item_n(it);
      const T* w = wire ? reinterpret_cast<const T*>(wire + it.meta_off) : nullptr;
      for (uint32_t e = lane_id(); e < n; e += 32) {
        float v = init_src ? __fmul_rn(DT<T>::to_float(init_src[it.elem_off + e]), prescale) : a[e];
        if (w) v = __fadd_rn(v, DT<T>::to_float(w[e]));
        a[e] = v;
      }
    }
  }
}

// The FP8 codecs of an 8-bit plan (the generic all-to-all, reduce-scatter and all-gather):
// wire = quantize(src * prescale), dst = decode(wire), acc (+)= decode(wire). Plain T tensors, round
// to nearest (the SR codecs: stochastically, with `rng`); the items are all compressed (the reducers
// pass raw layers to the max-min kernels). The SR codecs decode with their base format's kernels.
template <typename T, int CODEC, int GPL>
__global__ void __launch_bounds__(kThreads, 3)
quantize_items_fp8_kernel(const T* __restrict__ src, const WarpItem* __restrict__ items, uint32_t first,
                          uint32_t count, uint8_t* wire, float prescale, const RngKey rng) {
  const OneDst ds{wire};
  CGX_ITEM_LOOP(it) {
    const T* s = src + it.elem_off;
    if (item_kind(it) == kItemFull) {
      if (group_aligned<T>(s)) {
        float x[GPL][8];
        slice_load_vec<T, GPL>(s, x);
        slice_scale<GPL>(x, prescale);
        full_send_fp8_x<CODEC, GPL>(x, it, rng, ds);
      } else {
        full_send_fp8_scaled_unaligned<T, T, CODEC, GPL, false>(s, it, prescale, rng, ds, (T*)nullptr);
      }
    } else {
      bucket_send_fp8<T, T, CODEC>(s, it, prescale, rng, ds, (T*)nullptr);
    }
  }
}

template <typename T, int CODEC, int GPL>
__global__ void __launch_bounds__(kThreads, 3)
dequantize_items_fp8_kernel(const uint8_t* __restrict__ wire, const WarpItem* __restrict__ items, uint32_t first,
                            uint32_t count, T* __restrict__ dst) {
  CGX_ITEM_LOOP(it) {
    T* o = dst + it.elem_off;
    if (item_kind(it) == kItemFull) {
      if (group_aligned<T>(o)) {
        SliceWords<GPL> w;
        slice_fetch<8, GPL>(wire, it.meta_off, it.pay_off, item_lpb_log2(it), 8, w);
        full_recv_fp8_w<T, CODEC, GPL, true>(w, o);
      } else {
        full_recv_fp8_unaligned<T, CODEC, GPL>(wire, it, o);
      }
    } else {
      bucket_recv_fp8<T, CODEC>(wire, it, o);
    }
  }
}

// codes / scales = the records' FP8 codes and units, undecoded (the generic all-to-all's codes output)
template <int GPL>
__global__ void __launch_bounds__(kThreads, 3)
unpack_items_fp8_kernel(const uint8_t* __restrict__ wire, const WarpItem* __restrict__ items, uint32_t first,
                        uint32_t count, uint8_t* __restrict__ codes, float* __restrict__ scales, uint32_t bucket) {
  CGX_ITEM_LOOP(it) { fp8_unpack_item<GPL>(wire, it, codes + it.elem_off, scales + it.elem_off / bucket); }
}

// acc (fp32 scratch) = float(init_src) * prescale   (init_src != nullptr)
// acc = fl(acc + fl(float(code) * unit))            (wire != nullptr)
template <typename T, int CODEC, int GPL>
__global__ void __launch_bounds__(kThreads, 3)
accumulate_items_fp8_kernel(const uint8_t* __restrict__ wire, const WarpItem* __restrict__ items, uint32_t first,
                            uint32_t count, float* __restrict__ acc, uint32_t base_elem,
                            const T* __restrict__ init_src, float prescale) {
  const SrcSet ss{wire, 0u, 1, -1};
  CGX_ITEM_LOOP(it) {
    float* a = acc + (it.elem_off - base_elem);
    if (item_kind(it) == kItemFull) {
      float x[GPL][8];
      if (init_src) {
        slice_load_scalar<T, GPL>(init_src + it.elem_off, x);
        slice_scale<GPL>(x, prescale);
      } else {
        slice_load_scalar<float, GPL>(a, x);
      }
      if (wire) slice_accumulate_fp8<CODEC, GPL>(ss, it.meta_off, it.pay_off, item_lpb_log2(it), x);
      slice_store<float, GPL, false>(a, x);
    } else {
      const uint32_t n = item_n(it);
      const uint32_t ng = div_up(n, 8u);
      for (uint32_t g = lane_id(); g < ng; g += 32) {
        const int nv = (int)min(8u, n - g * 8u);
        float x[8];
        if (init_src) {
          load8_scalar<T>(init_src + it.elem_off + g * 8u, nv, x);
#pragma unroll
          for (int j = 0; j < 8; ++j) x[j] = __fmul_rn(x[j], prescale);
        } else {
          load8_scalar<float>(a + g * 8u, nv, x);
        }
        if (wire) bucket_add_sources_fp8<CODEC>(ss, it, g, x);
        store8_scalar<float>(a + g * 8u, nv, x);
      }
    }
  }
}

template <typename T>
__global__ void scale_kernel(T* __restrict__ data, uint64_t n, float scale) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    data[i] = DT<T>::from_float(__fmul_rn(DT<T>::to_float(data[i]), scale));
}

template <typename T>
__global__ void add_kernel(const T* __restrict__ x, const T* __restrict__ y, T* __restrict__ sum, uint64_t n) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    sum[i] = DT<T>::from_float(__fadd_rn(DT<T>::to_float(x[i]), DT<T>::to_float(y[i])));
}

template <typename TS, typename TD>
__global__ void convert_kernel(const TS* __restrict__ src, TD* __restrict__ dst, uint64_t n) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    dst[i] = DT<TD>::from_float(DT<TS>::to_float(src[i]));
}

int grid_for(uint32_t count) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const uint32_t want = (count + kWarps - 1) / kWarps;
  const uint32_t cap = (uint32_t)sms * 3u;  // one resident wave (3 CTAs of 8 warps per SM); warps loop
  return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}
int grid_for_elems(uint64_t n) {
  const uint64_t want = (n + 1023) / 1024;
  return (int)(want < 1 ? 1 : (want > 4096 ? 4096 : want));
}

// KB x GPL dispatch of a kernel template taking <..., KB, GPL>
#define CGX_DISPATCH_KB_GPL(a, CALL)                       \
  do {                                                     \
    const int kb_ = (a).uniform_bits;                      \
    if ((a).slice_elems == 1024) {                         \
      if (kb_ == 2) { CALL(2, 4); }                        \
      else if (kb_ == 4) { CALL(4, 4); }                   \
      else if (kb_ == 8) { CALL(8, 4); }                   \
      else { CALL(0, 4); }                                 \
    } else {                                               \
      if (kb_ == 2) { CALL(2, 2); }                        \
      else if (kb_ == 4) { CALL(4, 2); }                   \
      else if (kb_ == 8) { CALL(8, 2); }                   \
      else { CALL(0, 2); }                                 \
    }                                                      \
  } while (0)

template <typename TS, typename T>
cudaError_t quantize_t(const ItemKernelArgs& a, const TS* src, uint32_t base_elem, uint8_t* wire, float prescale,
                       const RngKey& rng, T* out, cudaStream_t stream) {
  if (a.count == 0) return cudaSuccess;
  const int grid = grid_for(a.count);
#define CGX_CALL(KB_, GPL_)                                                                                   \
  quantize_items_kernel<TS, T, KB_, GPL_><<<grid, kThreads, 0, stream>>>(src, base_elem, a.items, a.first, a.count, \
                                                                         wire, prescale, rng, out)
  CGX_DISPATCH_KB_GPL(a, CGX_CALL);
#undef CGX_CALL
  return cudaGetLastError();
}

template <typename T>
cudaError_t dequantize_t(const ItemKernelArgs& a, const uint8_t* wire, T* dst, cudaStream_t stream) {
  if (a.count == 0) return cudaSuccess;
  const int grid = grid_for(a.count);
#define CGX_CALL(KB_, GPL_) \
  dequantize_items_kernel<T, KB_, GPL_><<<grid, kThreads, 0, stream>>>(wire, a.items, a.first, a.count, dst)
  CGX_DISPATCH_KB_GPL(a, CGX_CALL);
#undef CGX_CALL
  return cudaGetLastError();
}

// CODEC x GPL dispatch of the FP8 kernels (8-bit plans only); the SR codecs only where the kernel
// encodes (SR: true)
#define CGX_DISPATCH_FP8_SR(a, SR, CALL)                           \
  do {                                                             \
    if ((a).uniform_bits != 8) return cudaErrorInvalidValue;       \
    const bool g4_ = (a).slice_elems == 1024;                      \
    const int c_ = (SR) ? (a).codec : fp8_base((a).codec);         \
    if (c_ == kE4M3) {                                             \
      if (g4_) { CALL(kE4M3, 4); } else { CALL(kE4M3, 2); }       \
    } else if (c_ == kE5M2) {                                      \
      if (g4_) { CALL(kE5M2, 4); } else { CALL(kE5M2, 2); }       \
    } else if (c_ == kE4M3Pow2) {                                  \
      if (g4_) { CALL(kE4M3Pow2, 4); } else { CALL(kE4M3Pow2, 2); } \
    } else if (c_ == kE5M2Pow2) {                                  \
      if (g4_) { CALL(kE5M2Pow2, 4); } else { CALL(kE5M2Pow2, 2); } \
    } else if ((SR) && c_ == kE4M3SR) {                            \
      if (g4_) { CALL(kE4M3SR, 4); } else { CALL(kE4M3SR, 2); }   \
    } else if ((SR) && c_ == kE5M2SR) {                            \
      if (g4_) { CALL(kE5M2SR, 4); } else { CALL(kE5M2SR, 2); }   \
    } else {                                                       \
      return cudaErrorInvalidValue;                                \
    }                                                              \
  } while (0)
#define CGX_DISPATCH_FP8(a, CALL) CGX_DISPATCH_FP8_SR(a, false, CALL)

template <typename T>
cudaError_t quantize_fp8_t(const ItemKernelArgs& a, const T* src, uint8_t* wire, float prescale, const RngKey& rng,
                           cudaStream_t stream) {
  if (a.count == 0) return cudaSuccess;
  const int grid = grid_for(a.count);
#define CGX_CALL(C_, GPL_)                                                                                      \
  quantize_items_fp8_kernel<T, C_, GPL_><<<grid, kThreads, 0, stream>>>(src, a.items, a.first, a.count, wire, prescale, \
                                                                        rng)
  CGX_DISPATCH_FP8_SR(a, true, CGX_CALL);
#undef CGX_CALL
  return cudaGetLastError();
}

template <typename T>
cudaError_t dequantize_fp8_t(const ItemKernelArgs& a, const uint8_t* wire, T* dst, cudaStream_t stream) {
  if (a.count == 0) return cudaSuccess;
  const int grid = grid_for(a.count);
#define CGX_CALL(C_, GPL_) \
  dequantize_items_fp8_kernel<T, C_, GPL_><<<grid, kThreads, 0, stream>>>(wire, a.items, a.first, a.count, dst)
  CGX_DISPATCH_FP8(a, CGX_CALL);
#undef CGX_CALL
  return cudaGetLastError();
}

template <typename T>
cudaError_t accumulate_fp8_t(const ItemKernelArgs& a, const uint8_t* wire, float* acc, uint32_t base_elem,
                             const T* init_src, float prescale, cudaStream_t stream) {
  if (a.count == 0) return cudaSuccess;
  const int grid = grid_for(a.count);
#define CGX_CALL(C_, GPL_)                                                                                \
  accumulate_items_fp8_kernel<T, C_, GPL_><<<grid, kThreads, 0, stream>>>(wire, a.items, a.first, a.count, acc, \
                                                                          base_elem, init_src, prescale)
  CGX_DISPATCH_FP8(a, CGX_CALL);
#undef CGX_CALL
  return cudaGetLastError();
}

template <typename T>
cudaError_t accumulate_t(const ItemKernelArgs& a, const uint8_t* wire, float* acc, uint32_t base_elem,
                         const T* init_src, float prescale, cudaStream_t stream) {
  if (a.count == 0) return cudaSuccess;
  const int grid = grid_for(a.count);
#define CGX_CALL(KB_, GPL_)                                                                                      \
  accumulate_items_kernel<T, KB_, GPL_><<<grid, kThreads, 0, stream>>>(wire, a.items, a.first, a.count, acc, base_elem, \
                                                                       init_src, prescale)
  CGX_DISPATCH_KB_GPL(a, CGX_CALL);
#undef CGX_CALL
  return cudaGetLastError();
}

}  // namespace

#define CGX_BY_DTYPE(dt, EXPR_F32, EXPR_F16, EXPR_BF16) \
  switch (dt) {                                         \
    case kF32: return EXPR_F32;                         \
    case kF16: return EXPR_F16;                         \
    case kBF16: return EXPR_BF16;                       \
    default: return cudaErrorInvalidValue;              \
  }

cudaError_t launch_quantize_items(const ItemKernelArgs& a, const void* src, uint8_t* wire, float prescale,
                                  const RngKey& rng, cudaStream_t stream) {
  if (a.codec != kMaxMin) {
    if (rng.enabled && !fp8_sr(a.codec)) return cudaErrorInvalidValue;
    CGX_BY_DTYPE(a.dtype, (quantize_fp8_t<float>(a, (const float*)src, wire, prescale, rng, stream)),
                 (quantize_fp8_t<__half>(a, (const __half*)src, wire, prescale, rng, stream)),
                 (quantize_fp8_t<__nv_bfloat16>(a, (const __nv_bfloat16*)src, wire, prescale, rng, stream)))
  }
  CGX_BY_DTYPE(a.dtype,
               (quantize_t<float, float>(a, (const float*)src, 0, wire, prescale, rng, nullptr, stream)),
               (quantize_t<__half, __half>(a, (const __half*)src, 0, wire, prescale, rng, nullptr, stream)),
               (quantize_t<__nv_bfloat16, __nv_bfloat16>(a, (const __nv_bfloat16*)src, 0, wire, prescale, rng, nullptr,
                                                         stream)))
}

cudaError_t launch_quantize_items_f32(const ItemKernelArgs& a, const float* src_f32, uint32_t base_elem,
                                      uint8_t* wire, const RngKey& rng, void* out, cudaStream_t stream) {
  if (a.codec != kMaxMin) {
    // the FP8 kernels of an fp32 tensor, on the scratch seen from the tensor's element 0 (items
    // address src + elem_off), then out = decode(wire)
    if (rng.enabled && !fp8_sr(a.codec)) return cudaErrorInvalidValue;
    cudaError_t e = quantize_fp8_t<float>(a, src_f32 - base_elem, wire, 1.0f, rng, stream);
    if (e != cudaSuccess || out == nullptr) return e;
    return launch_dequantize_items(a, wire, out, stream);
  }
  CGX_BY_DTYPE(a.dtype, (quantize_t<float, float>(a, src_f32, base_elem, wire, 1.0f, rng, (float*)out, stream)),
               (quantize_t<float, __half>(a, src_f32, base_elem, wire, 1.0f, rng, (__half*)out, stream)),
               (quantize_t<float, __nv_bfloat16>(a, src_f32, base_elem, wire, 1.0f, rng, (__nv_bfloat16*)out, stream)))
}

cudaError_t launch_dequantize_items(const ItemKernelArgs& a, const uint8_t* wire, void* dst, cudaStream_t stream) {
  if (a.codec != kMaxMin)
    CGX_BY_DTYPE(a.dtype, (dequantize_fp8_t<float>(a, wire, (float*)dst, stream)),
                 (dequantize_fp8_t<__half>(a, wire, (__half*)dst, stream)),
                 (dequantize_fp8_t<__nv_bfloat16>(a, wire, (__nv_bfloat16*)dst, stream)))
  CGX_BY_DTYPE(a.dtype, (dequantize_t<float>(a, wire, (float*)dst, stream)),
               (dequantize_t<__half>(a, wire, (__half*)dst, stream)),
               (dequantize_t<__nv_bfloat16>(a, wire, (__nv_bfloat16*)dst, stream)))
}

cudaError_t launch_unpack_items_fp8(const ItemKernelArgs& a, const uint8_t* wire, uint8_t* codes, float* scales,
                                    uint32_t bucket, cudaStream_t stream) {
  if (a.count == 0) return cudaSuccess;
  if (a.uniform_bits != 8 || bucket == 0) return cudaErrorInvalidValue;
  const int grid = grid_for(a.count);
  if (a.slice_elems == 1024)
    unpack_items_fp8_kernel<4><<<grid, kThreads, 0, stream>>>(wire, a.items, a.first, a.count, codes, scales, bucket);
  else
    unpack_items_fp8_kernel<2><<<grid, kThreads, 0, stream>>>(wire, a.items, a.first, a.count, codes, scales, bucket);
  return cudaGetLastError();
}

cudaError_t launch_accumulate_items_f32(const ItemKernelArgs& a, const uint8_t* wire, float* acc_f32,
                                        uint32_t base_elem, const void* init_src, float prescale,
                                        cudaStream_t stream) {
  if (a.codec != kMaxMin)
    CGX_BY_DTYPE(a.dtype,
                 (accumulate_fp8_t<float>(a, wire, acc_f32, base_elem, (const float*)init_src, prescale, stream)),
                 (accumulate_fp8_t<__half>(a, wire, acc_f32, base_elem, (const __half*)init_src, prescale, stream)),
                 (accumulate_fp8_t<__nv_bfloat16>(a, wire, acc_f32, base_elem, (const __nv_bfloat16*)init_src,
                                                  prescale, stream)))
  CGX_BY_DTYPE(a.dtype, (accumulate_t<float>(a, wire, acc_f32, base_elem, (const float*)init_src, prescale, stream)),
               (accumulate_t<__half>(a, wire, acc_f32, base_elem, (const __half*)init_src, prescale, stream)),
               (accumulate_t<__nv_bfloat16>(a, wire, acc_f32, base_elem, (const __nv_bfloat16*)init_src, prescale,
                                            stream)))
}

cudaError_t launch_scale_inplace(void* data, int dtype, uint64_t n, float scale, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const int grid = grid_for_elems(n);
  switch (dtype) {
    case kF32: scale_kernel<float><<<grid, 256, 0, stream>>>((float*)data, n, scale); break;
    case kF16: scale_kernel<__half><<<grid, 256, 0, stream>>>((__half*)data, n, scale); break;
    case kBF16: scale_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((__nv_bfloat16*)data, n, scale); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t launch_add(const void* x, const void* y, void* sum, int dtype, uint64_t n, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const int grid = grid_for_elems(n);
  switch (dtype) {
    case kF32: add_kernel<float><<<grid, 256, 0, stream>>>((const float*)x, (const float*)y, (float*)sum, n); break;
    case kF16: add_kernel<__half><<<grid, 256, 0, stream>>>((const __half*)x, (const __half*)y, (__half*)sum, n); break;
    case kBF16:
      add_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)y,
                                                         (__nv_bfloat16*)sum, n);
      break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t launch_convert(const void* src, int src_dtype, void* dst, int dst_dtype, uint64_t n, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const int grid = grid_for_elems(n);
#define CGX_CVT(TS_, TD_) convert_kernel<TS_, TD_><<<grid, 256, 0, stream>>>((const TS_*)src, (TD_*)dst, n)
  if (src_dtype == kF32 && dst_dtype == kF16) CGX_CVT(float, __half);
  else if (src_dtype == kF32 && dst_dtype == kBF16) CGX_CVT(float, __nv_bfloat16);
  else if (src_dtype == kF16 && dst_dtype == kF32) CGX_CVT(__half, float);
  else if (src_dtype == kBF16 && dst_dtype == kF32) CGX_CVT(__nv_bfloat16, float);
  else if (src_dtype == kF16 && dst_dtype == kBF16) CGX_CVT(__half, __nv_bfloat16);
  else if (src_dtype == kBF16 && dst_dtype == kF16) CGX_CVT(__nv_bfloat16, __half);
  else if (src_dtype == dst_dtype) return cudaMemcpyAsync(dst, src, n * (uint64_t)dtype_size(src_dtype), cudaMemcpyDeviceToDevice, stream);
  else return cudaErrorInvalidValue;
#undef CGX_CVT
  return cudaGetLastError();
}

}  // namespace cgx

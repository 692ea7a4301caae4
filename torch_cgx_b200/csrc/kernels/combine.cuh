// Weighted top-k combine of one token's slot rows (DESIGN §2.13d): the one function that does the
// arithmetic, called by the fused all-to-all's last arriver (a2a_kernel, COMBINE) and by the
// standalone combine_rows_kernel of the composed path, so both give the same bits.
#pragma once
#include <type_traits>
#include "device_utils.cuh"
#include "item_path.cuh"

namespace cgx {
namespace dev {

// one element through L2, as fp32
template <typename T>
__device__ __forceinline__ float ld_cg_float(const T* p) {
  if constexpr (sizeof(T) == 4) {
    return __ldcg(reinterpret_cast<const float*>(p));
  } else {
    const unsigned short b = __ldcg(reinterpret_cast<const unsigned short*>(p));
    if constexpr (std::is_same_v<T, __half>)
      return __half2float(__ushort_as_half(b));
    else
      return __uint_as_float((uint32_t)b << 16);  // bfloat16 -> fp32 is exact
  }
}

// Elements [0, n) of one segment, by the 32 lanes of a warp: slot0 is the segment's first element
// in slot row t * k (slot row t * k + c starts H elements further per c), g the token's k gates,
// out the segment's first element in the output row. For every element
//   acc = g_0 * x_0;  acc = fma(g_c, x_c, acc) for c = 1 .. k - 1;  out = T(acc), round to nearest,
// x_c the slot value in fp32. The slots are read through L2 (ld.global.cg): other SMs wrote them
// during the same launch.
template <typename T>
__device__ __forceinline__ void combine_segment(const T* slot0, uint64_t H, const float* __restrict__ g, uint32_t k,
                                                T* out, uint32_t n) {
  constexpr uint32_t V = (uint32_t)DT<T>::kVec;
  const uint32_t lane = lane_id();
  uint32_t done = 0;
  if (((reinterpret_cast<uintptr_t>(slot0) | reinterpret_cast<uintptr_t>(out) | (uintptr_t)(H * sizeof(T))) & 15u) ==
      0) {
    const uint32_t vecs = n / V;
    for (uint32_t v = lane; v < vecs; v += 32) {
      float acc[V], x[V];
      unpack16<T>(__ldcg(reinterpret_cast<const uint4*>(slot0) + v), acc);
      const float g0 = g[0];
#pragma unroll
      for (uint32_t i = 0; i < V; ++i) acc[i] = __fmul_rn(g0, acc[i]);
      for (uint32_t c = 1; c < k; ++c) {
        unpack16<T>(__ldcg(reinterpret_cast<const uint4*>(slot0 + c * H) + v), x);
        const float gc = g[c];
#pragma unroll
        for (uint32_t i = 0; i < V; ++i) acc[i] = __fmaf_rn(gc, x[i], acc[i]);
      }
      reinterpret_cast<uint4*>(out)[v] = pack16<T>(acc);
    }
    done = vecs * V;
  }
  for (uint32_t i = done + lane; i < n; i += 32) {
    float acc = __fmul_rn(g[0], ld_cg_float(slot0 + i));
    for (uint32_t c = 1; c < k; ++c) acc = __fmaf_rn(g[c], ld_cg_float(slot0 + c * H + i), acc);
    out[i] = DT<T>::from_float(acc);
  }
}

}  // namespace dev
}  // namespace cgx

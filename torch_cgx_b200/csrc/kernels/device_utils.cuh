// PTX-level helpers for sm_90a: system-scope flag signalling over NVLink,
// cache-bypassing vector loads of peer-written buffers, dtype conversion.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace cgx {
namespace dev {

// ---- dtype traits ----------------------------------------------------------
template <typename T>
struct DT;
template <>
struct DT<float> {
  static constexpr int kVec = 4;  // elements per 16 B
  __device__ __forceinline__ static float to_float(float v) { return v; }
  __device__ __forceinline__ static float from_float(float v) { return v; }
};
template <>
struct DT<__half> {
  static constexpr int kVec = 8;
  __device__ __forceinline__ static float to_float(__half v) { return __half2float(v); }
  __device__ __forceinline__ static __half from_float(float v) { return __float2half_rn(v); }
};
template <>
struct DT<__nv_bfloat16> {
  static constexpr int kVec = 8;
  __device__ __forceinline__ static float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ __forceinline__ static __nv_bfloat16 from_float(float v) { return __float2bfloat16_rn(v); }
};

// T(x * s): one fp32 multiply, rounded to nearest even in T (fp32: no second rounding); scale_round
// gives it back in fp32. The scaled send of the routed all-to-all (DESIGN §2.13e) sends these values.
template <typename T>
__device__ __forceinline__ T scale_round_to(float x, float s) {
  return DT<T>::from_float(__fmul_rn(x, s));
}
template <typename T>
__device__ __forceinline__ float scale_round(float x, float s) {
  return DT<T>::to_float(scale_round_to<T>(x, s));
}

// 16 B of T <-> fp32 registers
template <typename T>
__device__ __forceinline__ void unpack16(const uint4& raw, float* out);
template <>
__device__ __forceinline__ void unpack16<float>(const uint4& raw, float* out) {
  out[0] = __uint_as_float(raw.x);
  out[1] = __uint_as_float(raw.y);
  out[2] = __uint_as_float(raw.z);
  out[3] = __uint_as_float(raw.w);
}
template <>
__device__ __forceinline__ void unpack16<__half>(const uint4& raw, float* out) {
  const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __half22float2(h[i]);
    out[2 * i] = f.x;
    out[2 * i + 1] = f.y;
  }
}
template <>
__device__ __forceinline__ void unpack16<__nv_bfloat16>(const uint4& raw, float* out) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __bfloat1622float2(h[i]);
    out[2 * i] = f.x;
    out[2 * i + 1] = f.y;
  }
}
template <typename T>
__device__ __forceinline__ uint4 pack16(const float* in);
template <>
__device__ __forceinline__ uint4 pack16<float>(const float* in) {
  return make_uint4(__float_as_uint(in[0]), __float_as_uint(in[1]), __float_as_uint(in[2]),
                    __float_as_uint(in[3]));
}
template <>
__device__ __forceinline__ uint4 pack16<__half>(const float* in) {
  uint4 r;
  __half2* h = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(in[2 * i], in[2 * i + 1]);
  return r;
}
template <>
__device__ __forceinline__ uint4 pack16<__nv_bfloat16>(const float* in) {
  uint4 r;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(in[2 * i], in[2 * i + 1]);
  return r;
}

// ---- memory access ---------------------------------------------------------
// Buffers written by PEERS during the kernel (recv slots) must never be served
// from this SM's (non-coherent) L1: relaxed.sys loads go to L2, the point of
// coherence for NVLink writes into this GPU's memory.
__device__ __forceinline__ uint4 ld_sys_v4(const void* p) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ uint2 ld_sys_v2(const void* p) {
  uint2 v;
  asm volatile("ld.relaxed.sys.global.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_sys_u32(const void* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_sys_u16(const void* p) {
  uint16_t v;
  asm volatile("ld.relaxed.sys.global.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_sys_u8(const void* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// streaming load of this rank's own gradients (read exactly once)
__device__ __forceinline__ uint4 ld_stream_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
// store to a (possibly peer-mapped) global address
__device__ __forceinline__ void st_v4(void* p, const uint4& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// ---- cross-GPU signalling ---------------------------------------------------
// Release: all writes of the CTA that happened-before (bar.sync) the calling
// thread become visible system-wide before the flag value does.
__device__ __forceinline__ void st_release_sys(uint32_t* flag, uint32_t v) {
  asm volatile("fence.acq_rel.sys;\n\tst.relaxed.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* flag) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Spin until *flag reaches `epoch` (wrap-safe). Returns 0 when it did, 1 on timeout, 2 when the
// host asked every kernel of this heap to give up (`abort_word`, host-mapped memory, polled only
// every 1024 spins: it costs a PCIe round trip).
__device__ __forceinline__ int wait_flag(const uint32_t* flag, uint32_t epoch, uint64_t timeout_ns,
                                         const uint32_t* abort_word) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while ((int32_t)(ld_acquire_sys(flag) - epoch) < 0) {
    if ((++spins & 0x3FFu) == 0) {
      if (abort_word != nullptr && *reinterpret_cast<const volatile uint32_t*>(abort_word) != 0) return 2;
      uint64_t now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > timeout_ns) return 1;
    }
  }
  return 0;
}

}  // namespace dev
}  // namespace cgx

// Warp-item device primitives shared by every sm_90a kernel of the framework
// (fused SRA, one-shot, standalone quantize / dequantize / accumulate).
//
// One warp owns one *item* (common/wire.h) end to end in registers:
//   full item    a slice of 512 / 1024 elements made of whole power-of-two buckets.
//                Lane l holds the adjacent pack groups {l*GPL .. l*GPL+GPL-1} (8 consecutive
//                elements each, GPL = 2 or 4): two 128-bit loads per group for fp32, one 128-bit
//                load for fp16 / bf16; per-bucket min/max with FMNMX trees + redux.sync
//                (whole-slice buckets) or sub-warp butterflies (buckets 8..256); quantization
//                without a single F2I / I2F (levels live in the mantissa of 2^23 + q); shift-add
//                tree packing; the packed words of a lane are adjacent, so they leave as ONE
//                4/8/16-byte store per lane (128-512 contiguous bytes per warp instruction) to
//                peer memory, or as ONE multimem.st to the NVLS multicast mapping.
//   bucket item  any single bucket (partial tails, sizes that are not powers of two, > 1024):
//                generic predicated two-pass code, out of line.
//   raw items    uncompressed elements: classic two-shot allreduce, or in-switch reduction
//                with multimem.ld_reduce when the heap has a multicast mapping.
// Numerics are those of common/quant_math.h bit for bit (the CPU code is the oracle).
//
// Replaces the reference's three kernels per layer slice (find_meta, pack_array, UnpackArray:
// /root/reference/src/common/compression/cuda_compression_operations.cu:98-153, :287-371,
// :474-544) and its _add kernel (:58-65).
#pragma once
#include "../common/philox.h"
#include "../common/quant_math.h"
#include "../common/wire.h"
#include "device_utils.cuh"

namespace cgx {
namespace dev {

constexpr uint32_t kAll = 0xffffffffu;
constexpr uint32_t kMagicBits = 0x4B000000u;  // float bits of 2^23: 2^23 + q has q in its low mantissa bits
#define CGX_MAGIC 8388608.0f
#define CGX_INF_POS __int_as_float(0x7f800000)
#define CGX_INF_NEG __int_as_float(0xff800000)

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

// ---- where packed data goes ------------------------------------------------
// ONE destination: a plain (local or peer-mapped) pointer -- SRA phase A, staging, standalone kernels.
struct OneDst {
  uint8_t* p;  // base of the destination slot
};
// MANY destinations -- SRA phase B, one-shot phase 1: ONE multicast address (NVLS: the switch
// replicates the write into every rank's copy of the heap), or the same offset in `n`
// peer-mapped heaps (minus `skip`), plus an optional extra plain copy.
struct MultiDst {
  uint8_t* const* bases;  // [n] region bases (kernel parameter space)
  uint8_t* mc;            // multicast alias of the region, or nullptr
  uint32_t off;           // byte offset added to every base (slot of the writer)
  int n;
  int skip;               // index not to write (-1: none)
  uint8_t* local;         // additional plain store into this (local) region base, or nullptr
};

// Source set of a reduction: `n` slots of MY heap, `stride` bytes apart (minus `skip`).
struct SrcSet {
  const uint8_t* base;
  uint32_t stride;
  int n;
  int skip;
};

__device__ __forceinline__ void st_u32(void* p, uint32_t v) {
  asm volatile("st.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_u16(void* p, uint32_t v) {
  asm volatile("st.global.u16 [%0], %1;" ::"l"(p), "h"((uint16_t)v) : "memory");
}
__device__ __forceinline__ void st_u8(void* p, uint32_t v) {
  asm volatile("st.global.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_v2(void* p, uint32_t a, uint32_t b) {
  asm volatile("st.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
// NVLS stores: one instruction, the NVSwitch writes all replicas
__device__ __forceinline__ void mc_st_u32(void* p, uint32_t v) {
  asm volatile("multimem.st.relaxed.sys.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void mc_st_v2(void* p, uint32_t a, uint32_t b) {
  asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(__uint_as_float(a)),
               "f"(__uint_as_float(b))
               : "memory");
}
__device__ __forceinline__ void mc_st_v4(void* p, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
               : "memory");
}
// in-switch reduction of 16 B across every rank's copy (fp32 accumulation for 16-bit types)
template <typename T>
__device__ __forceinline__ uint4 mc_ld_reduce_v4(const void* p);
template <>
__device__ __forceinline__ uint4 mc_ld_reduce_v4<float>(const void* p) {
  float a, b, c, d;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(a), "=f"(b), "=f"(c), "=f"(d)
               : "l"(p)
               : "memory");
  return make_uint4(__float_as_uint(a), __float_as_uint(b), __float_as_uint(c), __float_as_uint(d));
}
template <>
__device__ __forceinline__ uint4 mc_ld_reduce_v4<__half>(const void* p) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
template <>
__device__ __forceinline__ uint4 mc_ld_reduce_v4<__nv_bfloat16>(const void* p) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

// (not unrolled: the bases come straight from the constant bank, one LDC per store; unrolling makes
// ptxas hoist W pointers into registers it does not have)
#define CGX_FOR_DST(ds, q)                         \
  _Pragma("unroll 1") for (int q = 0; q < (ds).n; ++q) \
    if (q != (ds).skip)

__device__ __forceinline__ void dst_st_u8(const OneDst& ds, uint32_t off, uint32_t v) { st_u8(ds.p + off, v); }
__device__ __forceinline__ void dst_st_u16(const OneDst& ds, uint32_t off, uint32_t v) { st_u16(ds.p + off, v); }
__device__ __forceinline__ void dst_st_u32(const OneDst& ds, uint32_t off, uint32_t v) { st_u32(ds.p + off, v); }
__device__ __forceinline__ void dst_st_v2(const OneDst& ds, uint32_t off, uint32_t a, uint32_t b) {
  st_v2(ds.p + off, a, b);
}
__device__ __forceinline__ void dst_st_v4(const OneDst& ds, uint32_t off, const uint4& v) { st_v4(ds.p + off, v); }

// sub-word stores have no multimem form: always through the unicast mappings
__device__ __forceinline__ void dst_st_u8(const MultiDst& ds, uint32_t off, uint32_t v) {
  CGX_FOR_DST(ds, q) st_u8(ds.bases[q] + ds.off + off, v);
  if (ds.local) st_u8(ds.local + ds.off + off, v);
}
__device__ __forceinline__ void dst_st_u16(const MultiDst& ds, uint32_t off, uint32_t v) {
  CGX_FOR_DST(ds, q) st_u16(ds.bases[q] + ds.off + off, v);
  if (ds.local) st_u16(ds.local + ds.off + off, v);
}
__device__ __forceinline__ void dst_st_u32(const MultiDst& ds, uint32_t off, uint32_t v) {
  if (ds.mc) {
    mc_st_u32(ds.mc + ds.off + off, v);
  } else {
    CGX_FOR_DST(ds, q) st_u32(ds.bases[q] + ds.off + off, v);
  }
  if (ds.local) st_u32(ds.local + ds.off + off, v);
}
__device__ __forceinline__ void dst_st_v2(const MultiDst& ds, uint32_t off, uint32_t a, uint32_t b) {
  if (ds.mc) {
    mc_st_v2(ds.mc + ds.off + off, a, b);
  } else {
    CGX_FOR_DST(ds, q) st_v2(ds.bases[q] + ds.off + off, a, b);
  }
  if (ds.local) st_v2(ds.local + ds.off + off, a, b);
}
__device__ __forceinline__ void dst_st_v4(const MultiDst& ds, uint32_t off, const uint4& v) {
  if (ds.mc) {
    mc_st_v4(ds.mc + ds.off + off, v);
  } else {
    CGX_FOR_DST(ds, q) st_v4(ds.bases[q] + ds.off + off, v);
  }
  if (ds.local) st_v4(ds.local + ds.off + off, v);
}
// the same destinations, unicast only (generic paths whose stores have no multimem form)
__device__ __forceinline__ OneDst unicast_of(const OneDst& ds) { return ds; }
__device__ __forceinline__ MultiDst unicast_of(const MultiDst& ds) {
  MultiDst d = ds;
  d.mc = nullptr;
  return d;
}

// ---- 8 elements <-> registers ---------------------------------------------------
// vector access needs (address % 32 == 0) for fp32 (two adjacent 128-bit LDG/STG) and % 16 for 16-bit types
template <typename T>
__device__ __forceinline__ bool group_aligned(const void* p) {
  return (reinterpret_cast<uintptr_t>(p) & (sizeof(T) * 8u - 1u)) == 0;
}

template <typename T>
__device__ __forceinline__ void load8_vec(const T* p, float (&x)[8]);
template <>
__device__ __forceinline__ void load8_vec<float>(const float* p, float (&x)[8]) {
  asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%8];\n\tld.global.v4.f32 {%4,%5,%6,%7}, [%8+16];"
               : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3]), "=f"(x[4]), "=f"(x[5]), "=f"(x[6]), "=f"(x[7])
               : "l"(p));
}
template <>
__device__ __forceinline__ void load8_vec<__half>(const __half* p, float (&x)[8]) {
  unpack16<__half>(*reinterpret_cast<const uint4*>(p), x);
}
template <>
__device__ __forceinline__ void load8_vec<__nv_bfloat16>(const __nv_bfloat16* p, float (&x)[8]) {
  unpack16<__nv_bfloat16>(*reinterpret_cast<const uint4*>(p), x);
}
// nv valid elements (0..8), the rest read as 0
template <typename T>
__device__ __forceinline__ void load8_scalar(const T* p, int nv, float (&x)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] = (j < nv) ? DT<T>::to_float(p[j]) : 0.f;
}

template <typename T>
__device__ __forceinline__ void store8_vec(T* p, const float (&x)[8]);
template <>
__device__ __forceinline__ void store8_vec<float>(float* p, const float (&x)[8]) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};\n\tst.global.v4.f32 [%0+16], {%5,%6,%7,%8};" ::"l"(p),
               "f"(x[0]), "f"(x[1]), "f"(x[2]),
               "f"(x[3]), "f"(x[4]), "f"(x[5]), "f"(x[6]), "f"(x[7])
               : "memory");
}
template <>
__device__ __forceinline__ void store8_vec<__half>(__half* p, const float (&x)[8]) {
  *reinterpret_cast<uint4*>(p) = pack16<__half>(x);
}
template <>
__device__ __forceinline__ void store8_vec<__nv_bfloat16>(__nv_bfloat16* p, const float (&x)[8]) {
  *reinterpret_cast<uint4*>(p) = pack16<__nv_bfloat16>(x);
}
template <typename T>
__device__ __forceinline__ void store8_scalar(T* p, int nv, const float (&x)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (j < nv) p[j] = DT<T>::from_float(x[j]);
}

// ---- min / max --------------------------------------------------------------------
// sm_90 has only the two-input min.NaN / max.NaN (FMNMX); the three-input form is sm_100+
__device__ __forceinline__ float min3_nan(float a, float b, float c) {
  float r;
  asm("{\n\t.reg .f32 t;\n\tmin.NaN.f32 t, %1, %2;\n\tmin.NaN.f32 %0, t, %3;\n\t}" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}
__device__ __forceinline__ float max3_nan(float a, float b, float c) {
  float r;
  asm("{\n\t.reg .f32 t;\n\tmax.NaN.f32 t, %1, %2;\n\tmax.NaN.f32 %0, t, %3;\n\t}" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}
__device__ __forceinline__ void minmax8(const float (&x)[8], float& mn, float& mx) {
  mn = min3_nan(min3_nan(min3_nan(x[0], x[1], x[2]), x[3], x[4]), min3_nan(x[5], x[6], x[7]), mn);
  mx = max3_nan(max3_nan(max3_nan(x[0], x[1], x[2]), x[3], x[4]), max3_nan(x[5], x[6], x[7]), mx);
}
__device__ __forceinline__ void minmax8_pred(const float (&x)[8], int nv, float& mn, float& mx) {
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (j < nv) {
      mn = nan_min(mn, x[j]);
      mx = nan_max(mx, x[j]);
    }
}

// Warp-wide min/max with one redux.sync each: floats are mapped to order-preserving signed
// integers (-0 < +0, like min.f32 / max.f32); NaN is handled by a vote so that it poisons the
// bucket exactly like the NaN-propagating scalar path of the CPU code.
__device__ __forceinline__ int float_to_ordered(float f) {
  const int b = __float_as_int(f);
  return b ^ ((b >> 31) & 0x7FFFFFFF);
}
__device__ __forceinline__ float ordered_to_float(int k) { return __int_as_float(k ^ ((k >> 31) & 0x7FFFFFFF)); }
__device__ __forceinline__ void warp_minmax(float& mn, float& mx) {
  const bool has_nan = __any_sync(kAll, (mn != mn) || (mx != mx));
  mn = ordered_to_float(__reduce_min_sync(kAll, float_to_ordered(mn)));
  mx = ordered_to_float(__reduce_max_sync(kAll, float_to_ordered(mx)));
  if (has_nan) mn = mx = __int_as_float(0x7fffffff);
}
// butterfly over aligned sub-groups of (1 << lg) lanes
__device__ __forceinline__ void subwarp_minmax(float& mn, float& mx, uint32_t lg) {
#pragma unroll
  for (uint32_t s = 0; s < 5; ++s) {
    if (s < lg) {
      mn = nan_min(mn, __shfl_xor_sync(kAll, mn, 1 << s));
      mx = nan_max(mx, __shfl_xor_sync(kAll, mx, 1 << s));
    }
  }
}

// ---- levels <-> packed words --------------------------------------------------------
// u = 2^23 + floor(t) for 0 <= t <= 255: the level is in the low mantissa bits, and
// (float)level == u - 2^23 exactly. No F2I / I2F on the hot path.
// CLAMP == false is only valid for deterministic rounding (r == 0.5) of a bucket whose min and
// max are finite: then 0.5 <= t < maxlvl + 1 and the clamp of encode_level() is a no-op.
template <bool CLAMP>
__device__ __forceinline__ float level_magic(float x, float mn, float inv, float r, float maxlvl) {
  float t = __fmaf_rn(__fsub_rn(x, mn), inv, r);
  if (CLAMP) t = fminf(t, maxlvl);  // NaN -> maxlvl, like encode_level()
  return __fadd_rz(t, CGX_MAGIC);
}

// Packing of 8 magic floats into a word: shift-adds in a depth-3 tree (7 IMADs, no masking);
// the 0x4B000000 of every term adds up to a constant that is subtracted once.
template <int KB>
__device__ __forceinline__ void pack_magic(const float (&u)[8], int bits, uint32_t& lo, uint32_t& hi) {
  if constexpr (KB >= 1 && KB <= 4) {
    uint32_t a[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) a[j] = (__float_as_uint(u[2 * j + 1]) << KB) + __float_as_uint(u[2 * j]);
    const uint32_t b0 = (a[1] << (2 * KB)) + a[0], b1 = (a[3] << (2 * KB)) + a[2];
    const uint32_t w = (b1 << (4 * KB)) + b0;
    // sum_j (0x4B000000 << 4j) mod 2^32 for KB == 4; for narrower words the magic bits never reach
    // the low 8*KB bits
    if constexpr (KB == 4)
      lo = w - 0xFB000000u;
    else
      lo = w & ((1u << (8 * KB)) - 1u);
    hi = 0;
  } else if constexpr (KB == 8) {
    const uint32_t a0 = (__float_as_uint(u[1]) << 8) + __float_as_uint(u[0]);
    const uint32_t a1 = (__float_as_uint(u[3]) << 8) + __float_as_uint(u[2]);
    const uint32_t a2 = (__float_as_uint(u[5]) << 8) + __float_as_uint(u[4]);
    const uint32_t a3 = (__float_as_uint(u[7]) << 8) + __float_as_uint(u[6]);
    lo = ((a1 << 16) + a0) - kMagicBits;
    hi = ((a3 << 16) + a2) - kMagicBits;
  } else {
    uint64_t w = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) w |= (uint64_t)(__float_as_uint(u[j]) & 0xFFu) << (j * bits);
    lo = (uint32_t)w;
    hi = (uint32_t)(w >> 32);
  }
}

// packed word -> 8 levels as floats
template <int KB>
__device__ __forceinline__ void unpack_magic(uint32_t lo, uint32_t hi, int bits, float (&qf)[8]) {
  if constexpr (KB == 8) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      qf[j] = __uint_as_float(__byte_perm(lo, kMagicBits, 0x7440 + j)) - CGX_MAGIC;
      qf[4 + j] = __uint_as_float(__byte_perm(hi, kMagicBits, 0x7440 + j)) - CGX_MAGIC;
    }
  } else if constexpr (KB == 4) {
    const uint32_t e = lo & 0x0F0F0F0Fu, o = (lo >> 4) & 0x0F0F0F0Fu;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      qf[2 * j] = __uint_as_float(__byte_perm(e, kMagicBits, 0x7440 + j)) - CGX_MAGIC;
      qf[2 * j + 1] = __uint_as_float(__byte_perm(o, kMagicBits, 0x7440 + j)) - CGX_MAGIC;
    }
  } else if constexpr (KB == 2) {
#pragma unroll
    for (int j = 0; j < 8; ++j) qf[j] = __uint_as_float(((lo >> (2 * j)) & 3u) | kMagicBits) - CGX_MAGIC;
  } else {
    const uint64_t w = (uint64_t)lo | ((uint64_t)hi << 32);
    const uint32_t mask = (1u << bits) - 1u;
#pragma unroll
    for (int j = 0; j < 8; ++j) qf[j] = __uint_as_float(((uint32_t)(w >> (j * bits)) & mask) | kMagicBits) - CGX_MAGIC;
  }
}

// load the packed word of group g from a (peer-written) payload
template <int KB>
__device__ __forceinline__ void load_word(const uint8_t* pay, uint32_t g, int bits, uint32_t& lo, uint32_t& hi) {
  hi = 0;
  if constexpr (KB == 8) {
    const uint2 v = ld_sys_v2(pay + (size_t)g * 8u);
    lo = v.x;
    hi = v.y;
  } else if constexpr (KB == 4) {
    lo = ld_sys_u32(pay + (size_t)g * 4u);
  } else if constexpr (KB == 2) {
    lo = ld_sys_u16(pay + (size_t)g * 2u);
  } else {
    const uint8_t* p = pay + (size_t)g * bits;
    uint64_t w = 0;
    for (int t = 0; t < bits; ++t) w |= (uint64_t)ld_sys_u8(p + t) << (8 * t);
    lo = (uint32_t)w;
    hi = (uint32_t)(w >> 32);
  }
}

// ---- a lane's words: lane l of the warp owns GPL *adjacent* pack groups (l*GPL .. l*GPL+GPL-1), so
// its packed words are GPL*KB contiguous bytes: one 4/8/16-byte access per lane, 128-512 contiguous
// bytes per warp instruction (large NVLink / multimem transactions instead of 4-byte ones).
template <int KB, int GPL>
__device__ __forceinline__ void load_words(const uint8_t* pay, int bits, uint32_t (&lo)[GPL], uint32_t (&hi)[GPL]) {
  const uint32_t g0 = lane_id() * GPL;
#pragma unroll
  for (int k = 0; k < GPL; ++k) hi[k] = 0;
  if constexpr (KB == 4 && GPL == 2) {
    const uint2 v = ld_sys_v2(pay + (size_t)g0 * 4u);
    lo[0] = v.x;
    lo[1] = v.y;
  } else if constexpr (KB == 8 && GPL == 2) {
    const uint4 v = ld_sys_v4(pay + (size_t)g0 * 8u);
    lo[0] = v.x, hi[0] = v.y, lo[1] = v.z, hi[1] = v.w;
  } else if constexpr (KB == 2 && GPL == 2) {
    const uint32_t v = ld_sys_u32(pay + (size_t)g0 * 2u);
    lo[0] = v & 0xFFFFu;
    lo[1] = v >> 16;
  } else if constexpr (KB == 4 && GPL == 4) {
    const uint4 v = ld_sys_v4(pay + (size_t)g0 * 4u);
    lo[0] = v.x, lo[1] = v.y, lo[2] = v.z, lo[3] = v.w;
  } else if constexpr (KB == 8 && GPL == 4) {
    const uint4 a = ld_sys_v4(pay + (size_t)g0 * 8u), b = ld_sys_v4(pay + (size_t)g0 * 8u + 16u);
    lo[0] = a.x, hi[0] = a.y, lo[1] = a.z, hi[1] = a.w, lo[2] = b.x, hi[2] = b.y, lo[3] = b.z, hi[3] = b.w;
  } else if constexpr (KB == 2 && GPL == 4) {
    const uint2 v = ld_sys_v2(pay + (size_t)g0 * 2u);
    lo[0] = v.x & 0xFFFFu, lo[1] = v.x >> 16, lo[2] = v.y & 0xFFFFu, lo[3] = v.y >> 16;
  } else {
#pragma unroll
    for (int k = 0; k < GPL; ++k) load_word<0>(pay, g0 + (uint32_t)k, bits, lo[k], hi[k]);
  }
}

template <int KB, int GPL, typename DST>
__device__ __forceinline__ void store_words(const DST& ds, uint32_t pay_off, int bits, const uint32_t (&lo)[GPL],
                                            const uint32_t (&hi)[GPL]) {
  const uint32_t g0 = lane_id() * GPL;
  if constexpr (KB == 4 && GPL == 2) {
    dst_st_v2(ds, pay_off + g0 * 4u, lo[0], lo[1]);
  } else if constexpr (KB == 8 && GPL == 2) {
    dst_st_v4(ds, pay_off + g0 * 8u, make_uint4(lo[0], hi[0], lo[1], hi[1]));
  } else if constexpr (KB == 2 && GPL == 2) {
    dst_st_u32(ds, pay_off + g0 * 2u, lo[0] | (lo[1] << 16));
  } else if constexpr (KB == 4 && GPL == 4) {
    dst_st_v4(ds, pay_off + g0 * 4u, make_uint4(lo[0], lo[1], lo[2], lo[3]));
  } else if constexpr (KB == 8 && GPL == 4) {
    dst_st_v4(ds, pay_off + g0 * 8u, make_uint4(lo[0], hi[0], lo[1], hi[1]));
    dst_st_v4(ds, pay_off + g0 * 8u + 16u, make_uint4(lo[2], hi[2], lo[3], hi[3]));
  } else if constexpr (KB == 2 && GPL == 4) {
    dst_st_v2(ds, pay_off + g0 * 2u, lo[0] | (lo[1] << 16), lo[2] | (lo[3] << 16));
  } else {
    // other widths: byte stores through the unicast mappings (the host never hands out a multicast
    // alias for plans with such widths)
#pragma unroll
    for (int k = 0; k < GPL; ++k) {
      const uint64_t w = (uint64_t)lo[k] | ((uint64_t)hi[k] << 32);
      const uint32_t o = pay_off + (g0 + (uint32_t)k) * (uint32_t)bits;
      for (int t = 0; t < bits; ++t) dst_st_u8(ds, o + t, (uint32_t)(w >> (8 * t)) & 0xFFu);
    }
  }
}

// the Philox word of one group (host twin: rounding_bits). The keys are made opaque per call:
// otherwise the ten round keys become loop invariants that the compiler hoists out of the item
// loops -- 18 registers the deterministic path needs.
__device__ __forceinline__ Philox4 rounding_word(const RngKey& rng, uint32_t first_elem) {
  uint32_t k0 = rng.seed_lo ^ (rng.stream * 0x9E3779B9u), k1 = rng.seed_hi;
  asm volatile("" : "+r"(k0), "+r"(k1));
  return philox4x32_10(first_elem, 0u, 0u, rng.seq, k0, k1);
}
// stochastic rounding offsets of one group from its Philox word (host twin: rounding_from_bits)
__device__ __forceinline__ void rounding8(const RngKey& rng, uint32_t first_elem, float (&r)[8]) {
  const Philox4 a = rounding_word(rng, first_elem);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t h = (a.v[j >> 1] >> ((j & 1) * 16)) & 0xFFFFu;
    r[j] = __uint_as_float(0x3F800000u | (h << 7)) - 1.0f;  // == h * 2^-16 exactly
  }
}

}  // namespace dev
}  // namespace cgx

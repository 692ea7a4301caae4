// Max-min uniform quantization numerics, shared verbatim by the CPU
// implementation and every CUDA kernel (host+device inline functions), so the
// CPU path is a bit-exact oracle for the GPU path.
//
// Behavioural spec (what, not how) follows the reference:
//   /root/reference/src/common/compression/cuda_compression_operations.cu:68-96
//   (encode/decode), :98-153 (per-bucket max/min -> unit), SURVEY.md §2.7.
// Deliberate differences: all arithmetic is fp32 regardless of the tensor
// dtype (the reference compares/accumulates fp16 in fp16), meta is stored as
// fp32, NaN/Inf propagate to the whole bucket instead of being dropped.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define CGX_HD __host__ __device__ __forceinline__
#else
#define CGX_HD inline
#endif

namespace cgx {

constexpr float kQuantEps = 1e-10f;  // unit below this => all levels are 0
constexpr int kPackGroup = 8;        // values per packed group (-> `bits` bytes)
constexpr int kRawBits = 32;         // "bits" value that means: do not compress

struct BucketMeta {
  float unit;
  float min;
};

// The GPU's canonical NaN: what every fp32 arithmetic instruction and min.NaN / max.NaN
// return when the result is NaN. The host code returns it too wherever a NaN can reach the
// wire, so that wire bytes of a poisoned bucket are identical on the CPU and the GPU (x86
// would keep the input's payload, or make 0xFFC00000 out of inf - inf).
constexpr uint32_t kCanonicalNaNBits = 0x7FFFFFFFu;
CGX_HD float canonical_nan() {
#if defined(__CUDA_ARCH__)
  return __int_as_float((int)kCanonicalNaNBits);
#else
  float f;
  std::memcpy(&f, &kCanonicalNaNBits, 4);
  return f;
#endif
}

// NaN-propagating min/max (a NaN gradient must poison its bucket so that AMP
// overflow checks on the reduced gradient still fire on every rank).
CGX_HD float nan_min(float a, float b) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
#else
  if (a != a || b != b) return canonical_nan();
  if (a == b) return std::signbit(a) ? a : b;  // -0 < +0, as PTX min does
  return a < b ? a : b;
#endif
}
CGX_HD float nan_max(float a, float b) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
#else
  if (a != a || b != b) return canonical_nan();
  if (a == b) return std::signbit(a) ? b : a;  // +0 > -0, as PTX max does
  return a > b ? a : b;
#endif
}

CGX_HD uint32_t max_level(int bits) { return (1u << bits) - 1u; }

// 1 / (2^bits - 1), correctly rounded to fp32 (a literal per width so that host and
// device agree bit for bit and the device pays one FMUL instead of an IEEE division)
CGX_HD float rcp_levels(int bits) {
  switch (bits) {
    case 1: return 1.0f;
    case 2: return 1.0f / 3.0f;
    case 3: return 1.0f / 7.0f;
    case 4: return 1.0f / 15.0f;
    case 5: return 1.0f / 31.0f;
    case 6: return 1.0f / 63.0f;
    case 7: return 1.0f / 127.0f;
    default: return 1.0f / 255.0f;
  }
}

// unit = (max - min) * fp32(1 / levels): one rounding for the difference, one for the product
CGX_HD BucketMeta make_meta(float mn, float mx, int bits) {
  BucketMeta m;
#if defined(__CUDA_ARCH__)
  m.unit = __fmul_rn(__fsub_rn(mx, mn), rcp_levels(bits));
#else
  m.unit = (mx - mn) * rcp_levels(bits);
  if (m.unit != m.unit) m.unit = canonical_nan();  // NaN min/max, or inf - inf
#endif
  m.min = mn;
  return m;
}

// 1/unit, or 0 when the bucket is (numerically) constant: every level is then
// 0 and the bucket decodes to `min` exactly (the property the reference's
// exactness test relies on, /root/reference/test/test_cgx.py:69-78).
CGX_HD float inv_unit(float unit) {
#if defined(__CUDA_ARCH__)
  return unit < kQuantEps ? 0.f : __frcp_rn(unit);  // correctly rounded == 1.0f / unit
#else
  return unit < kQuantEps ? 0.f : 1.0f / unit;
#endif
}

// level = clamp(floor((x - min) * inv + r), 0, maxlvl); r = 0.5 for
// deterministic rounding, U[0,1) for QSGD-style stochastic rounding.
CGX_HD uint32_t encode_level(float x, float mn, float inv, float r, float maxlvl_f) {
#if defined(__CUDA_ARCH__)
  float t = __fmaf_rn(__fsub_rn(x, mn), inv, r);
#else
  float t = std::fmaf(x - mn, inv, r);
#endif
  // t >= 0 always (x >= min, inv >= 0, r >= 0) unless it is NaN; fminf returns the
  // non-NaN operand on host and device, so NaN -> maxlvl.
  t = fminf(t, maxlvl_f);
  return (uint32_t)t;  // truncation == floor for t >= 0
}

CGX_HD float decode_level(uint32_t q, float unit, float mn) {
#if defined(__CUDA_ARCH__)
  return __fmaf_rn(unit, (float)q, mn);
#else
  return std::fmaf(unit, (float)q, mn);
#endif
}

// Pack 8 levels (each < 2^bits) into the low 8*bits bits of a 64-bit word,
// value j at bit j*bits; the word is emitted little-endian as `bits` bytes.
CGX_HD uint64_t pack8(const uint32_t q[8], int bits) {
  uint64_t w = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) w |= (uint64_t)q[j] << (j * bits);
  return w;
}
CGX_HD uint32_t unpack1(uint64_t w, int j, int bits) {
  return (uint32_t)(w >> (j * bits)) & ((1u << bits) - 1u);
}

}  // namespace cgx

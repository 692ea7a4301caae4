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
#include <type_traits>

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

// ---- FP8 wire codec (compressed all-to-all only) ---------------------------------------------
// What the bytes of an 8-bit record mean. kMaxMin: levels of [min, max] (above). kE4M3 / kE5M2:
// one fp32 scale per bucket, unit = max|x| * fp32(1 / FMAX), and one FP8 code per element,
// code = cvt.rn.satfinite(x * (1 / unit)), decoded as float(code) * unit. The record keeps the
// 8-bit layout: meta {unit, +0.0f} where max-min stores {unit, min}, then one byte per element.
// A NaN or an Inf in a bucket makes unit NaN or Inf and every element decodes to NaN (0 * Inf is
// NaN); a bucket whose unit is below 2^-126 has 1 / unit = 0 and decodes to signed zeros.
// kE4M3Pow2 / kE5M2Pow2: the element format of kE4M3 / kE5M2 with a power-of-two unit 2^k, k the
// smallest integer >= -126 with max|x| <= FMAX * 2^k (DESIGN §2.13g). x * 2^-k and code * 2^k are
// exact, so decode(encode(.)) is a projection, and every finite unit is an E8M0 value. A NaN or Inf
// bucket keeps unit = max|x| and decodes to NaN; a zero bucket has unit 2^-126.
// kE4M3SR / kE5M2SR: the records, units and decoder of kE4M3 / kE5M2; only the encoder differs, it
// rounds stochastically (fp8_sr_snap, DESIGN §2.13h) with the max-min encoder's random bits.
enum WireCodec : int { kMaxMin = 0, kE4M3 = 1, kE5M2 = 2, kE4M3Pow2 = 3, kE5M2Pow2 = 4, kE4M3SR = 5, kE5M2SR = 6 };

// the element format of an FP8 codec (kE4M3 or kE5M2), whether its units are powers of two, and
// whether it rounds stochastically; constant-folded where the codec is a template argument
CGX_HD constexpr int fp8_base(int codec) {
  return (codec == kE4M3Pow2 || codec == kE4M3SR) ? kE4M3 : (codec == kE5M2Pow2 || codec == kE5M2SR) ? kE5M2 : codec;
}
CGX_HD constexpr bool fp8_pow2(int codec) { return codec == kE4M3Pow2 || codec == kE5M2Pow2; }
CGX_HD constexpr bool fp8_sr(int codec) { return codec == kE4M3SR || codec == kE5M2SR; }
CGX_HD constexpr bool is_fp8_codec(int codec) { return codec >= kE4M3 && codec <= kE5M2SR; }

// f(std::integral_constant<int, C>()) for the FP8 codec C equal to `codec`, `otherwise` for any other
// value: how the launchers turn the runtime codec into the kernels' compile-time one
template <typename R, typename F>
R dispatch_fp8(int codec, R otherwise, F&& f) {
  switch (codec) {
    case kE4M3: return f(std::integral_constant<int, kE4M3>());
    case kE5M2: return f(std::integral_constant<int, kE5M2>());
    case kE4M3Pow2: return f(std::integral_constant<int, kE4M3Pow2>());
    case kE5M2Pow2: return f(std::integral_constant<int, kE5M2Pow2>());
    case kE4M3SR: return f(std::integral_constant<int, kE4M3SR>());
    case kE5M2SR: return f(std::integral_constant<int, kE5M2SR>());
    default: return otherwise;
  }
}

constexpr float kFp8MinUnit = 1.17549435e-38f;  // 2^-126: a smaller unit decodes its bucket to zeros
constexpr uint32_t kFp8NaNCode = 0x7Fu;         // the code cvt.rn.satfinite writes for any NaN

CGX_HD uint32_t fp32_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t u;
  std::memcpy(&u, &f, 4);
  return u;
#endif
}
CGX_HD float fp32_from_bits(uint32_t u) {
#if defined(__CUDA_ARCH__)
  return __uint_as_float(u);
#else
  float f;
  std::memcpy(&f, &u, 4);
  return f;
#endif
}

// largest finite value of the format, and its reciprocal correctly rounded to fp32 (a literal per
// format, as rcp_levels)
CGX_HD float fp8_max(int codec) { return fp8_base(codec) == kE5M2 ? 57344.0f : 448.0f; }
CGX_HD float fp8_rcp_max(int codec) { return fp8_base(codec) == kE5M2 ? 1.0f / 57344.0f : 1.0f / 448.0f; }

// the power-of-two unit of a bucket whose nan_max(-min, max) is a (a >= +0 or NaN). FMAX is
// 1.75 * 2^E (E = 8 for e4m3, 15 for e5m2), so for a = 1.f * 2^e, a <= FMAX * 2^k holds from
// k = e - E on when 1.f <= 1.75 (f <= 0x600000) and from e - E + 1 otherwise. Zeros and fp32
// subnormals give k < -126 and take the clamp. Integer operations only: no log2 / exp2 rounding.
CGX_HD float fp8_pow2_unit(float a, int codec) {
  const uint32_t ax = fp32_bits(a) & 0x7FFFFFFFu;
  if (ax >= 0x7F800000u) return a;  // NaN or +Inf: the bucket decodes to NaN, as with an fp32 unit
  const int E = fp8_base(codec) == kE5M2 ? 15 : 8;
  int k = (int)(ax >> 23) - 127 - E + ((ax & 0x7FFFFFu) > 0x600000u ? 1 : 0);
  k = k < -126 ? -126 : k;  // k <= 127 - 8 + 1 = 120: FLT_MAX <= 448 * 2^120
  return fp32_from_bits((uint32_t)(k + 127) << 23);
}

// steps 1-2: unit = nan_max(-min, max) * fp32(1 / FMAX), one rounding (the pow2 codecs: the unit of
// fp8_pow2_unit); the meta's second word is +0
CGX_HD BucketMeta fp8_meta(float mn, float mx, int codec) {
  BucketMeta m;
  const float a = nan_max(-mn, mx);
  if (fp8_pow2(codec)) {
    m.unit = fp8_pow2_unit(a, codec);
  } else {
#if defined(__CUDA_ARCH__)
    m.unit = __fmul_rn(a, fp8_rcp_max(codec));
#else
    m.unit = a * fp8_rcp_max(codec);
    if (m.unit != m.unit) m.unit = canonical_nan();
#endif
  }
  m.min = 0.f;
  return m;
}

// step 3: 1 / unit, or 0 below 2^-126 (NaN stays NaN: NaN < x is false). A finite pow2 unit 2^k
// (k in [-126, 120]) has the exact inverse 2^-k, exponent field 254 - (k + 127); NaN and Inf take
// the fp32-scale rule, so a poisoned bucket has the same codes in both formats.
CGX_HD float fp8_inv_unit(float unit, int codec) {
  if (fp8_pow2(codec) && fp32_bits(unit) < 0x7F800000u) return fp32_from_bits((254u - (fp32_bits(unit) >> 23)) << 23);
#if defined(__CUDA_ARCH__)
  return unit < kFp8MinUnit ? 0.f : __frcp_rn(unit);
#else
  return unit < kFp8MinUnit ? 0.f : 1.0f / unit;
#endif
}

// Software cvt.rn.satfinite.{e4m3,e5m2}.f32 of one value: round to nearest even on the format's grid
// (subnormals included), anything beyond the largest finite value -- infinities too -- saturates to
// it, and a NaN of any sign or payload becomes kFp8NaNCode.
inline uint32_t fp8_from_float_host(float v, int codec) {
  codec = fp8_base(codec);
  const int mb = codec == kE5M2 ? 2 : 3, bias = codec == kE5M2 ? 15 : 7;
  const uint32_t maxcode = codec == kE5M2 ? 0x7Bu : 0x7Eu;
  uint32_t u;
  std::memcpy(&u, &v, 4);
  const uint32_t sign = (u >> 24) & 0x80u, ax = u & 0x7FFFFFFFu;
  if (ax > 0x7F800000u) return kFp8NaNCode;
  const int e = (int)(ax >> 23) - 127;
  if (e == -127) return sign;  // zero or an fp32 subnormal: far below half the smallest FP8 subnormal
  const uint32_t man = (ax & 0x7FFFFFu) | 0x800000u;
  const int emin = 1 - bias;
  const int shift = 23 - mb + (e < emin ? emin - e : 0);
  if (shift > 24) return sign;  // below half the smallest subnormal
  uint32_t q = man >> shift;
  const uint32_t rem = man & ((1u << shift) - 1u), half = 1u << (shift - 1);
  if (rem > half || (rem == half && (q & 1u))) ++q;
  // a subnormal that rounds up to 2^mb, or a mantissa that rounds over, carries into the exponent
  uint32_t code = e < emin ? q : ((uint32_t)(e + bias) << mb) + q - (1u << mb);
  if (code > maxcode) code = maxcode;
  return sign | code;
}

// exact value of an FP8 code
inline float fp8_to_float_host(uint32_t code, int codec) {
  codec = fp8_base(codec);
  const int mb = codec == kE5M2 ? 2 : 3, bias = codec == kE5M2 ? 15 : 7;
  const uint32_t mag = code & 0x7Fu, ef = mag >> mb, mf = mag & ((1u << mb) - 1u);
  float v;
  if (codec == kE5M2 ? ef == 0x1Fu : mag == 0x7Fu)
    v = (codec == kE5M2 && mf == 0) ? INFINITY : canonical_nan();
  else if (ef == 0)
    v = std::ldexp((float)mf, 1 - bias - mb);
  else
    v = std::ldexp((float)(mf | (1u << mb)), (int)ef - bias - mb);
  return (code & 0x80u) ? -v : v;
}

// cvt.rn.satfinite of two values already in the format's units: the code of a in bits 0..7, of b
// in bits 8..15 (the order of the 8-bit record). cvt's first source goes to the upper byte.
CGX_HD uint32_t fp8x2_cvt(float a, float b, int codec) {
#if defined(__CUDA_ARCH__)
  unsigned short h;
  if (fp8_base(codec) == kE5M2)
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(h) : "f"(b), "f"(a));
  else
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(h) : "f"(b), "f"(a));
  return h;
#else
  return fp8_from_float_host(a, codec) | (fp8_from_float_host(b, codec) << 8);
#endif
}

// steps 4-5 for two elements, the unit the device converts
CGX_HD uint32_t fp8x2_encode(float x0, float x1, float inv, int codec) {
#if defined(__CUDA_ARCH__)
  return fp8x2_cvt(__fmul_rn(x0, inv), __fmul_rn(x1, inv), codec);
#else
  return fp8x2_cvt(x0 * inv, x1 * inv, codec);
#endif
}

// Stochastic rounding of y = fp32(x * inv) onto the format's grid (kE4M3SR / kE5M2SR, DESIGN §2.13h),
// with h the element's 16 random bits: the grid spacing at |y| is s = 2^(max(e, emin) - mb), t = |y| / s
// = n + f, and |y| becomes (n + 1) * s iff h + floor(2^16 * f) >= 2^16, else n * s: floor(t + h * 2^-16),
// the rule encode_level applies to max-min levels. The result is y's sign times that grid value, which
// cvt.rn.satfinite then converts exactly (or saturates); NaN and Inf pass unchanged (-> the NaN code,
// FMAX), and fp32 subnormals become +-0. Integer operations on the bits of y only, the same on host and
// device. t's discarded bits are those below bit `shift` of the mantissa with its implicit bit.
CGX_HD float fp8_sr_snap(float y, uint32_t h, int codec) {
  const int mb = fp8_base(codec) == kE5M2 ? 2 : 3, emin_b = fp8_base(codec) == kE5M2 ? 127 - 14 : 127 - 6;
  const uint32_t u = fp32_bits(y), ay = u & 0x7FFFFFFFu, eb = ay >> 23;
  if (ay >= 0x7F800000u) return y;
  const uint32_t shift = 23u - (uint32_t)mb + ((int)eb < emin_b ? (uint32_t)(emin_b - (int)eb) : 0u);
  const uint32_t man = (ay & 0x7FFFFFu) | 0x800000u;
  // d >= 4, and floor(2^16 f) = (man mod 2^shift) >> d; man < 2^24, so it is 0 once d >= 24: zeros
  // and fp32 subnormals (shift > 100) round to 0
  const uint32_t d = shift - 16u;
  const uint32_t f16 = (man >> (d < 31u ? d : 31u)) & 0xFFFFu;
  const uint32_t up = ((h & 0xFFFFu) + f16) >> 16;
  uint32_t r;
  if (shift <= 23u)
    r = (ay & ~((1u << shift) - 1u)) + (up << shift);  // n * s, plus s: a carry into the exponent is exact
  else
    r = up ? (uint32_t)(emin_b - mb) << 23 : 0u;  // n = 0: 0 or s, the format's smallest subnormal
  return fp32_from_bits((u & 0x80000000u) | r);
}

// two elements of an SR codec, with the random bits of each
CGX_HD uint32_t fp8x2_encode_sr(float x0, float x1, float inv, int codec, uint32_t h0, uint32_t h1) {
#if defined(__CUDA_ARCH__)
  const float a = __fmul_rn(x0, inv), b = __fmul_rn(x1, inv);
#else
  const float a = x0 * inv, b = x1 * inv;
#endif
  return fp8x2_cvt(fp8_sr_snap(a, h0, codec), fp8_sr_snap(b, h1, codec), codec);
}
CGX_HD void fp8x2_decode(uint32_t pair, float unit, int codec, float& d0, float& d1) {
#if defined(__CUDA_ARCH__)
  const unsigned short in = (unsigned short)pair;
  uint32_t h2;
  if (fp8_base(codec) == kE5M2)
    asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(h2) : "h"(in));
  else
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(in));
  float f0, f1;
  asm("{\n\t.reg .b16 lo, hi;\n\tmov.b32 {lo, hi}, %2;\n\tcvt.f32.f16 %0, lo;\n\tcvt.f32.f16 %1, hi;\n\t}"
      : "=f"(f0), "=f"(f1)
      : "r"(h2));
  d0 = __fmul_rn(f0, unit);
  d1 = __fmul_rn(f1, unit);
#else
  d0 = fp8_to_float_host(pair & 0xFFu, codec) * unit;
  d1 = fp8_to_float_host((pair >> 8) & 0xFFu, codec) * unit;
  if (d0 != d0) d0 = canonical_nan();
  if (d1 != d1) d1 = canonical_nan();
#endif
}

// one element (the host codec and the generic paths)
CGX_HD uint32_t fp8_encode(float x, float inv, int codec) { return fp8x2_encode(x, 0.f, inv, codec) & 0xFFu; }
CGX_HD uint32_t fp8_encode_sr(float x, float inv, int codec, uint32_t h) {
  return fp8x2_encode_sr(x, 0.f, inv, codec, h, 0u) & 0xFFu;
}
CGX_HD float fp8_decode(uint32_t code, float unit, int codec) {
  float d0, d1;
  fp8x2_decode(code & 0xFFu, unit, codec, d0, d1);
  return d0;
}

}  // namespace cgx

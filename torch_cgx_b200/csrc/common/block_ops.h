// Host (CPU) implementation of the four block primitives every reducer is
// built from: load (+prescale), quantize, decode-accumulate, decode-store.
// Same arithmetic as the CUDA kernels (quant_math.h / philox.h), so it serves
// as (1) the CPU-tensor path of the backend and (2) the bit-exact oracle the
// GPU tests compare against.
//
// Role in the reference: MaxMinQuantizer::CompressBuffer/DecompressBuffer and
// DummyCompressor (/root/reference/src/common/compressor.cc:222-253,301-399),
// Compressor::Add (:196-205).
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>
#include "philox.h"
#include "quant_math.h"
#include "wire.h"

namespace cgx {
namespace cpu {

// ---- software fp16 / bf16 (round-to-nearest-even, matches __float2half_rn /
// __float2bfloat16_rn) ------------------------------------------------------
inline float bits_to_float(uint32_t u) {
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}
inline uint32_t float_to_bits(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  return u;
}
inline float half_to_float(uint16_t h) {
  uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1Fu;
  uint32_t man = h & 0x3FFu;
  if (exp == 0) {
    if (man == 0) return bits_to_float(sign);
    // subnormal: value = man * 2^-24
    float f = (float)man * (1.0f / 16777216.0f);
    return (sign ? -f : f);
  }
  if (exp == 31) return bits_to_float(sign | 0x7F800000u | (man << 13));
  return bits_to_float(sign | ((exp + 112u) << 23) | (man << 13));
}
inline uint16_t float_to_half(float f) {
  uint32_t x = float_to_bits(f);
  uint32_t sign = (x >> 16) & 0x8000u;
  uint32_t ax = x & 0x7FFFFFFFu;
  if (ax >= 0x7F800000u) {  // inf / nan
    return (uint16_t)(sign | 0x7C00u | (ax > 0x7F800000u ? 0x200u | ((ax >> 13) & 0x3FFu) : 0u));
  }
  if (ax >= 0x477FF000u) return (uint16_t)(sign | 0x7C00u);  // rounds to >= 65520 -> inf
  if (ax < 0x33000001u) return (uint16_t)sign;               // < 2^-25 (or == 2^-25 ties to 0)
  int32_t e = (int32_t)(ax >> 23) - 127;
  uint32_t man = (ax & 0x7FFFFFu) | 0x800000u;
  if (e < -14) {
    // subnormal half: shift so that the result is man * 2^(e+24) with 10-bit precision
    int shift = -14 - e + 13;  // 14..24
    uint32_t q = man >> shift;
    uint32_t rem = man & ((1u << shift) - 1u);
    uint32_t half = 1u << (shift - 1);
    if (rem > half || (rem == half && (q & 1u))) ++q;
    return (uint16_t)(sign | q);
  }
  uint32_t q = ((uint32_t)(e + 15) << 10) | ((man >> 13) & 0x3FFu);
  uint32_t rem = man & 0x1FFFu;
  if (rem > 0x1000u || (rem == 0x1000u && (q & 1u))) ++q;  // carry may bump the exponent: correct
  return (uint16_t)(sign | q);
}
inline float bf16_to_float(uint16_t h) { return bits_to_float((uint32_t)h << 16); }
inline uint16_t float_to_bf16(float f) {
  uint32_t x = float_to_bits(f);
  if ((x & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)((x >> 16) | 0x40u);  // quiet NaN
  uint32_t lsb = (x >> 16) & 1u;
  x += 0x7FFFu + lsb;
  return (uint16_t)(x >> 16);
}

inline float load_elem(const void* base, int dtype, uint64_t i) {
  switch (dtype) {
    case kF32: return ((const float*)base)[i];
    case kF16: return half_to_float(((const uint16_t*)base)[i]);
    default: return bf16_to_float(((const uint16_t*)base)[i]);
  }
}
inline void store_elem(void* base, int dtype, uint64_t i, float v) {
  switch (dtype) {
    case kF32: ((float*)base)[i] = v; break;
    case kF16: ((uint16_t*)base)[i] = float_to_half(v); break;
    default: ((uint16_t*)base)[i] = float_to_bf16(v); break;
  }
}
// value as it will be seen after a store+load round trip in `dtype`
inline float round_to_dtype(float v, int dtype) {
  switch (dtype) {
    case kF32: return v;
    case kF16: return half_to_float(float_to_half(v));
    default: return bf16_to_float(float_to_bf16(v));
  }
}

// acc[i] = float(src[elem_off + i]) * prescale; a NaN product is the GPU's canonical NaN, as it is
// on the device (raw records carry these values on the wire)
inline void load_block(const void* src, int dtype, const BlockDesc& d, float prescale, float* acc) {
  const uint32_t n = block_n(d);
  for (uint32_t i = 0; i < n; ++i) {
    const float v = load_elem(src, dtype, (uint64_t)d.elem_off + i) * prescale;
    acc[i] = v == v ? v : canonical_nan();
  }
}

// Quantize n fp32 values into the block's wire record. Buckets are self-contained: bucket k
// owns meta[k] and the pack groups [k * bucket_groups(B), ...) of the payload.
inline void quantize_block(const float* acc, int dtype, const BlockDesc& d, uint8_t* rec,
                           const RngKey& rng, uint32_t /*block_id*/) {
  const uint32_t n = block_n(d);
  const int bits = block_bits(d);
  if (bits >= kRawBits) {
    for (uint32_t i = 0; i < n; ++i) store_elem(rec, dtype, i, acc[i]);
    uint32_t used = n * (uint32_t)dtype_size(dtype), tot = align_up(used, kWireAlign);
    std::memset(rec + used, 0, tot - used);
    return;
  }
  const uint32_t B = d.bucket;
  const uint32_t nb = block_num_buckets(n, B);
  const uint32_t gpb = bucket_groups(B);
  BucketMeta* meta = reinterpret_cast<BucketMeta*>(rec);
  uint8_t* pay = rec + block_meta_bytes(n, B);
  const float maxlvl = (float)max_level(bits);
  for (uint32_t b = 0; b < nb; ++b) {
    const uint32_t lo = b * B, hi = lo + B < n ? lo + B : n;
    float mn = acc[lo], mx = acc[lo];
    for (uint32_t i = lo + 1; i < hi; ++i) {
      mn = nan_min(mn, acc[i]);
      mx = nan_max(mx, acc[i]);
    }
    meta[b] = make_meta(mn, mx, bits);
    const float inv = inv_unit(meta[b].unit);
    const uint32_t groups = div_up(hi - lo, 8u);
    for (uint32_t g = 0; g < groups; ++g) {
      const uint32_t i0 = lo + g * 8u;
      float r[8];
      rounding_offsets8(rng, d.elem_off + i0, r);
      uint32_t q[8];
      for (int j = 0; j < 8; ++j) q[j] = (i0 + j < hi) ? encode_level(acc[i0 + j], meta[b].min, inv, r[j], maxlvl) : 0u;
      const uint64_t w = pack8(q, bits);
      uint8_t* dst = pay + (size_t)(b * gpb + g) * bits;
      for (int t = 0; t < bits; ++t) dst[t] = (uint8_t)(w >> (8 * t));
    }
  }
  {
    uint32_t used = nb * 8u, tot = block_meta_bytes(n, B);
    std::memset(rec + used, 0, tot - used);
  }
  {
    uint32_t used = block_num_groups(n, B) * (uint32_t)bits, tot = block_payload_bytes(n, bits, B);
    std::memset(pay + used, 0, tot - used);
  }
}

// Decode element i of a block record to fp32 (already rounded to `dtype` for
// raw blocks, exact fp32 for quantized ones).
template <typename F>
inline void decode_block_foreach(const uint8_t* rec, int dtype, const BlockDesc& d, F&& f) {
  const uint32_t n = block_n(d);
  const int bits = block_bits(d);
  if (bits >= kRawBits) {
    for (uint32_t i = 0; i < n; ++i) f(i, load_elem(rec, dtype, i));
    return;
  }
  const uint32_t B = d.bucket;
  const uint32_t nb = block_num_buckets(n, B);
  const uint32_t gpb = bucket_groups(B);
  const BucketMeta* meta = reinterpret_cast<const BucketMeta*>(rec);
  const uint8_t* pay = rec + block_meta_bytes(n, B);
  for (uint32_t b = 0; b < nb; ++b) {
    const uint32_t lo = b * B, hi = lo + B < n ? lo + B : n;
    const BucketMeta m = meta[b];
    const uint32_t groups = div_up(hi - lo, 8u);
    for (uint32_t g = 0; g < groups; ++g) {
      const uint8_t* src = pay + (size_t)(b * gpb + g) * bits;
      uint64_t w = 0;
      for (int t = 0; t < bits; ++t) w |= (uint64_t)src[t] << (8 * t);
      for (int j = 0; j < 8; ++j) {
        const uint32_t i = lo + g * 8u + (uint32_t)j;
        if (i >= hi) break;
        f(i, decode_level(unpack1(w, j, bits), m.unit, m.min));
      }
    }
  }
}

// FP8 codecs (quant_math.h) of an 8-bit block: the record layout of quantize_block at bits 8,
// meta {unit, +0} per bucket and element i's code at byte i of its bucket's payload. The SR codecs
// draw element j of the pack group at block element i0 from half j of rounding_bits(rng, elem_off + i0),
// the bits the max-min encoder would use for it; the others ignore rng.
inline void quantize_block_fp8(const float* acc, const BlockDesc& d, uint8_t* rec, int codec, const RngKey& rng) {
  const uint32_t n = block_n(d);
  const uint32_t B = d.bucket;
  const uint32_t nb = block_num_buckets(n, B);
  const uint32_t gpb = bucket_groups(B);
  BucketMeta* meta = reinterpret_cast<BucketMeta*>(rec);
  uint8_t* pay = rec + block_meta_bytes(n, B);
  for (uint32_t b = 0; b < nb; ++b) {
    const uint32_t lo = b * B, hi = lo + B < n ? lo + B : n;
    float mn = acc[lo], mx = acc[lo];
    for (uint32_t i = lo + 1; i < hi; ++i) {
      mn = nan_min(mn, acc[i]);
      mx = nan_max(mx, acc[i]);
    }
    meta[b] = fp8_meta(mn, mx, codec);
    const float inv = fp8_inv_unit(meta[b].unit, codec);
    uint8_t* dst = pay + (size_t)b * gpb * 8u;
    if (fp8_sr(codec)) {
      for (uint32_t i0 = lo; i0 < hi; i0 += 8u) {
        const Philox4 a = rounding_bits(rng, d.elem_off + i0);
        for (uint32_t j = 0; j < 8u; ++j)
          dst[i0 - lo + j] = i0 + j < hi ? (uint8_t)fp8_encode_sr(acc[i0 + j], inv, codec, a.v[j >> 1] >> ((j & 1u) * 16u)) : 0u;
      }
      continue;
    }
    for (uint32_t i = lo; i < lo + div_up(hi - lo, 8u) * 8u; ++i)
      dst[i - lo] = i < hi ? (uint8_t)fp8_encode(acc[i], inv, codec) : 0u;
  }
  {
    uint32_t used = nb * 8u, tot = block_meta_bytes(n, B);
    std::memset(rec + used, 0, tot - used);
  }
  {
    uint32_t used = block_num_groups(n, B) * 8u, tot = block_payload_bytes(n, 8, B);
    std::memset(pay + used, 0, tot - used);
  }
}

inline void decode_block_fp8_store(const uint8_t* rec, int dtype, const BlockDesc& d, void* dst, int codec) {
  const uint32_t n = block_n(d);
  const uint32_t B = d.bucket;
  const uint32_t nb = block_num_buckets(n, B);
  const uint32_t gpb = bucket_groups(B);
  const BucketMeta* meta = reinterpret_cast<const BucketMeta*>(rec);
  const uint8_t* pay = rec + block_meta_bytes(n, B);
  for (uint32_t b = 0; b < nb; ++b) {
    const uint32_t lo = b * B, hi = lo + B < n ? lo + B : n;
    const uint8_t* src = pay + (size_t)b * gpb * 8u;
    for (uint32_t i = lo; i < hi; ++i)
      store_elem(dst, dtype, (uint64_t)d.elem_off + i, fp8_decode(src[i - lo], meta[b].unit, codec));
  }
}

// An FP8 record undecoded (the all-to-all's codes output): codes[elem_off + i] = element i's code,
// scales[(elem_off + i) / B] = its bucket's unit; elem_off is a multiple of B
inline void unpack_block_fp8(const uint8_t* rec, const BlockDesc& d, uint8_t* codes, float* scales) {
  const uint32_t n = block_n(d);
  const uint32_t B = d.bucket;
  const uint32_t nb = block_num_buckets(n, B);
  const uint32_t gpb = bucket_groups(B);
  const BucketMeta* meta = reinterpret_cast<const BucketMeta*>(rec);
  const uint8_t* pay = rec + block_meta_bytes(n, B);
  for (uint32_t b = 0; b < nb; ++b) {
    const uint32_t lo = b * B, hi = lo + B < n ? lo + B : n;
    scales[d.elem_off / B + b] = meta[b].unit;
    std::memcpy(codes + (size_t)d.elem_off + lo, pay + (size_t)b * gpb * 8u, hi - lo);
  }
}

// acc[i] = fl(acc[i] + fl(float(code) * unit)): the reduce-scatter's accumulation of an FP8 record
inline void decode_block_fp8_add(const uint8_t* rec, const BlockDesc& d, float* acc, int codec) {
  const uint32_t n = block_n(d);
  const uint32_t B = d.bucket;
  const uint32_t nb = block_num_buckets(n, B);
  const uint32_t gpb = bucket_groups(B);
  const BucketMeta* meta = reinterpret_cast<const BucketMeta*>(rec);
  const uint8_t* pay = rec + block_meta_bytes(n, B);
  for (uint32_t b = 0; b < nb; ++b) {
    const uint32_t lo = b * B, hi = lo + B < n ? lo + B : n;
    const uint8_t* src = pay + (size_t)b * gpb * 8u;
    for (uint32_t i = lo; i < hi; ++i) {
      const float v = acc[i] + fp8_decode(src[i - lo], meta[b].unit, codec);
      acc[i] = v == v ? v : canonical_nan();
    }
  }
}

inline void decode_block_add(const uint8_t* rec, int dtype, const BlockDesc& d, float* acc) {
  decode_block_foreach(rec, dtype, d, [&](uint32_t i, float v) { acc[i] += v; });
}

inline void decode_block_store(const uint8_t* rec, int dtype, const BlockDesc& d, void* dst) {
  decode_block_foreach(rec, dtype, d,
                       [&](uint32_t i, float v) { store_elem(dst, dtype, (uint64_t)d.elem_off + i, v); });
}

}  // namespace cpu
}  // namespace cgx

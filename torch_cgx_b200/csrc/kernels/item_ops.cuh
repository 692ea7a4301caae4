// Item-level operations built from item_path.cuh. Each function is executed by ONE warp on ONE
// item. The hot versions work on a slice whose values are already in registers (the callers
// prefetch the next item's data while the current one is processed) and assume 16/32 B aligned
// gradients; everything rare -- unaligned slices, generic buckets, raw tails -- is deliberately
// out of line so that the hot loops stay a few hundred instructions long.
//
//   *_send     quantize my values of an item and store the packed words to a destination
//              (SRA phase A, one-shot phase 1, standalone quantize)
//   *_reduce   own values + the decoded copies of W-1 sources, requantize, publish, self-decode
//              (SRA phase B)
//   *_recv     decode one source -- or the sum of all sources -- into the gradient buffer
//              (SRA phase C, one-shot phase 2, standalone dequantize)
// Reference counterparts: Compressor::Compress / Decompress per layer slice
// (/root/reference/src/common/compressor.cc:98-179) and the SRA loop bodies
// (/root/reference/src/common/scatter_reduce_allgather.cc:116-199).
#pragma once
#include "item_path.cuh"

namespace cgx {
namespace dev {

template <int GPL>
struct SliceCfg {
  static constexpr uint32_t kElems = 256u * GPL;
  static constexpr uint32_t kLgAll = GPL == 4 ? 7u : 6u;  // log2(bucket/8) of a bucket spanning the slice
  static constexpr int kPeerBatch = 2;  // sources fetched before any is consumed
};

// one bucket == the whole slice (512 / 1024-element buckets): the common case
template <int GPL>
__device__ __forceinline__ bool slice_single_bucket(uint32_t lg) {
  return GPL == 4 || lg == SliceCfg<GPL>::kLgAll;
}

// ---- slice <-> registers -------------------------------------------------------------
// Lane l owns the GPL adjacent pack groups l*GPL .. l*GPL+GPL-1, i.e. GPL*8 consecutive elements
// (row k of the register tile = group l*GPL + k). Its packed words are then adjacent too.
template <int GPL>
__device__ __forceinline__ uint32_t lane_group(int k) {
  return lane_id() * GPL + (uint32_t)k;
}
// issue the (vector) loads of a slice; `src` must be group aligned
template <typename TS, int GPL>
__device__ __forceinline__ void slice_load_vec(const TS* __restrict__ src, float (&x)[GPL][8]) {
  const TS* p = src + lane_id() * (GPL * 8u);
#pragma unroll
  for (int k = 0; k < GPL; ++k) load8_vec<TS>(p + k * 8, x[k]);
}
template <typename TS, int GPL>
__device__ __forceinline__ void slice_load_scalar(const TS* __restrict__ src, float (&x)[GPL][8]) {
  const TS* p = src + lane_id() * (GPL * 8u);
#pragma unroll
  for (int k = 0; k < GPL; ++k) load8_scalar<TS>(p + k * 8, 8, x[k]);
}
// pull the slice towards L2 without occupying registers (phase B prefetches its next item this way:
// its registers are taken by the peers' words)
template <typename TS, int GPL>
__device__ __forceinline__ void slice_prefetch_l2(const TS* __restrict__ src) {
  const TS* p = src + lane_id() * (GPL * 8u);
#pragma unroll
  for (int k = 0; k < GPL; ++k) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + k * 8));
}
template <int GPL>
__device__ __forceinline__ void slice_scale(float (&x)[GPL][8], float prescale) {
  if (prescale != 1.0f) {
#pragma unroll
    for (int k = 0; k < GPL; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) x[k][j] = __fmul_rn(x[k][j], prescale);
  }
}
template <typename TO, int GPL, bool VEC>
__device__ __forceinline__ void slice_store(TO* __restrict__ dst, const float (&x)[GPL][8]) {
  TO* p = dst + lane_id() * (GPL * 8u);
#pragma unroll
  for (int k = 0; k < GPL; ++k) {
    if (VEC)
      store8_vec<TO>(p + k * 8, x[k]);
    else
      store8_scalar<TO>(p + k * 8, 8, x[k]);
  }
}

// per-bucket {unit, min} and 1/unit of every group row of the slice
template <int GPL>
__device__ __forceinline__ void slice_meta(const float (&x)[GPL][8], uint32_t lg, int bits, BucketMeta (&m)[GPL],
                                           float (&inv)[GPL]) {
  float mn[GPL], mx[GPL];
#pragma unroll
  for (int k = 0; k < GPL; ++k) {
    mn[k] = CGX_INF_POS;
    mx[k] = CGX_INF_NEG;
    minmax8(x[k], mn[k], mx[k]);
  }
  if (slice_single_bucket<GPL>(lg)) {
    float a = mn[0], b = mx[0];
#pragma unroll
    for (int k = 1; k < GPL; ++k) {
      a = nan_min(a, mn[k]);
      b = nan_max(b, mx[k]);
    }
    warp_minmax(a, b);
    const BucketMeta m0 = make_meta(a, b, bits);
    const float i0 = inv_unit(m0.unit);
#pragma unroll
    for (int k = 0; k < GPL; ++k) {
      m[k] = m0;
      inv[k] = i0;
    }
  } else if (lg == 0) {  // 8-element buckets: every row is its own bucket
#pragma unroll
    for (int k = 0; k < GPL; ++k) {
      m[k] = make_meta(mn[k], mx[k], bits);
      inv[k] = inv_unit(m[k].unit);
    }
  } else {
    // (512-slices only) a bucket of 2^lg groups = all rows of 2^(lg-1) adjacent lanes
    float a = mn[0], b = mx[0];
#pragma unroll
    for (int k = 1; k < GPL; ++k) {
      a = nan_min(a, mn[k]);
      b = nan_max(b, mx[k]);
    }
    subwarp_minmax(a, b, lg - 1u);
    const BucketMeta m0 = make_meta(a, b, bits);
    const float i0 = inv_unit(m0.unit);
#pragma unroll
    for (int k = 0; k < GPL; ++k) {
      m[k] = m0;
      inv[k] = i0;
    }
  }
}

template <int GPL, typename DST>
__device__ __forceinline__ void slice_store_meta(const BucketMeta (&m)[GPL], uint32_t lg, const DST& ds,
                                                 uint32_t meta_off) {
  if (slice_single_bucket<GPL>(lg)) {
    if (lane_id() == 0) dst_st_v2(ds, meta_off, __float_as_uint(m[0].unit), __float_as_uint(m[0].min));
  } else {
#pragma unroll
    for (int k = 0; k < GPL; ++k) {
      const uint32_t gi = lane_group<GPL>(k);
      if ((gi & ((1u << lg) - 1u)) == 0)
        dst_st_v2(ds, meta_off + (gi >> lg) * 8u, __float_as_uint(m[k].unit), __float_as_uint(m[k].min));
    }
  }
}

// quantize + pack + store the slice; SELF: also write the decoded values (what every receiver
// will decode from the same bytes) to `self_out` (VEC: it is group aligned).
// MODE 0: deterministic rounding, every bucket finite (no clamp needed)  1: deterministic  2: stochastic
template <typename TO, int KB, int GPL, bool SELF, bool VEC, int MODE, typename DST>
__device__ __forceinline__ void slice_encode_mode(const float (&x)[GPL][8], const BucketMeta (&m)[GPL],
                                                  const float (&inv)[GPL], int bits, const RngKey& rng,
                                                  uint32_t first_elem, const DST& ds, uint32_t pay_off,
                                                  TO* __restrict__ self_out) {
  const float maxlvl = (float)max_level(bits);
  uint32_t lo[GPL], hi[GPL];
#pragma unroll
  for (int k = 0; k < GPL; ++k) {
    const uint32_t gi = lane_group<GPL>(k);
    float u[8];
    if (MODE == 2) {
      float r[8];
      rounding8(rng, first_elem + gi * 8u, r);
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = level_magic<true>(x[k][j], m[k].min, inv[k], r[j], maxlvl);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = level_magic<MODE == 1>(x[k][j], m[k].min, inv[k], 0.5f, maxlvl);
    }
    pack_magic<KB>(u, bits, lo[k], hi[k]);
    if (SELF) {
      float dec[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) dec[j] = __fmaf_rn(m[k].unit, __fsub_rn(u[j], CGX_MAGIC), m[k].min);
      if (VEC)
        store8_vec<TO>(self_out + gi * 8u, dec);
      else
        store8_scalar<TO>(self_out + gi * 8u, 8, dec);
    }
  }
  store_words<KB, GPL>(ds, pay_off, bits, lo, hi);
}

template <typename TO, int KB, int GPL, bool SELF, bool VEC, typename DST>
__device__ __forceinline__ void slice_encode(const float (&x)[GPL][8], const BucketMeta (&m)[GPL],
                                             const float (&inv)[GPL], int bits, const RngKey& rng,
                                             uint32_t first_elem, const DST& ds, uint32_t pay_off,
                                             TO* __restrict__ self_out) {
  if (rng.enabled) {
    slice_encode_mode<TO, KB, GPL, SELF, VEC, 2>(x, m, inv, bits, rng, first_elem, ds, pay_off, self_out);
    return;
  }
  // every bucket of the slice has finite min/max (unit finite <=> max - min finite) -> no clamp
  bool finite = true;
#pragma unroll
  for (int k = 0; k < GPL; ++k) finite = finite && (fabsf(m[k].unit) < CGX_INF_POS);
  if (__all_sync(kAll, finite))
    slice_encode_mode<TO, KB, GPL, SELF, VEC, 0>(x, m, inv, bits, rng, first_elem, ds, pay_off, self_out);
  else
    slice_encode_mode<TO, KB, GPL, SELF, VEC, 1>(x, m, inv, bits, rng, first_elem, ds, pay_off, self_out);
}

// packed words + meta of one source for a slice, as loaded (not yet decoded)
template <int GPL>
struct SliceWords {
  uint32_t lo[GPL], hi[GPL];
  BucketMeta pm[GPL];
};

// issue the loads of one source's packed words + meta for the slice (no use yet)
template <int KB, int GPL>
__device__ __forceinline__ void slice_fetch(const uint8_t* rec, uint32_t meta_off, uint32_t pay_off, uint32_t lg,
                                            int bits, SliceWords<GPL>& w) {
  load_words<KB, GPL>(rec + pay_off, bits, w.lo, w.hi);
  if (slice_single_bucket<GPL>(lg)) {
    const uint2 v = ld_sys_v2(rec + meta_off);
#pragma unroll
    for (int k = 0; k < GPL; ++k) {
      w.pm[k].unit = __uint_as_float(v.x);
      w.pm[k].min = __uint_as_float(v.y);
    }
  } else {
#pragma unroll
    for (int k = 0; k < GPL; ++k) {
      const uint2 v = ld_sys_v2(rec + meta_off + ((lane_group<GPL>(k) >> lg) * 8u));
      w.pm[k].unit = __uint_as_float(v.x);
      w.pm[k].min = __uint_as_float(v.y);
    }
  }
}

// x (+)= decode(words)
template <int KB, int GPL, bool ADD>
__device__ __forceinline__ void slice_decode(const SliceWords<GPL>& w, int bits, float (&x)[GPL][8]) {
#pragma unroll
  for (int k = 0; k < GPL; ++k) {
    float qf[8];
    unpack_magic<KB>(w.lo[k], w.hi[k], bits, qf);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = __fmaf_rn(w.pm[k].unit, qf[j], w.pm[k].min);
      x[k][j] = ADD ? __fadd_rn(x[k][j], d) : d;
    }
  }
}

// x += decode(source i) for every source of the set, in slot order.
// Common case (one bucket == the slice): ONE {unit, min} per source, so the words of up to 8
// sources are in flight at once -- at W = 8 the whole reduction of an item is a single round trip
// to L2/HBM instead of four dependent ones. Slices made of several small buckets keep a
// per-row meta and go two sources at a time.
template <int KB, int GPL>
__device__ __forceinline__ void slice_accumulate(const SrcSet& ss, uint32_t meta_off, uint32_t pay_off, uint32_t lg,
                                                 int bits, float (&x)[GPL][8]) {
  const int cnt = ss.n - (ss.skip >= 0 ? 1 : 0);
  if (slice_single_bucket<GPL>(lg)) {
    constexpr int kB = GPL == 4 ? 2 : 4;
    for (int i0 = 0; i0 < cnt; i0 += kB) {
      uint32_t lo[kB][GPL], hi[kB][GPL];
      float un[kB], mi[kB];
#pragma unroll
      for (int u = 0; u < kB; ++u) {
        // past the end: re-read the last source (unconditional loads keep the arrays in
        // registers; the value is simply not added)
        const int i = min(i0 + u, cnt - 1);
        const int q = (ss.skip >= 0 && i >= ss.skip) ? i + 1 : i;
        const uint8_t* rec = ss.base + (size_t)q * ss.stride;
        load_words<KB, GPL>(rec + pay_off, bits, lo[u], hi[u]);
        const uint2 v = ld_sys_v2(rec + meta_off);
        un[u] = __uint_as_float(v.x);
        mi[u] = __uint_as_float(v.y);
      }
#pragma unroll
      for (int u = 0; u < kB; ++u) {
        if (i0 + u < cnt) {
#pragma unroll
          for (int k = 0; k < GPL; ++k) {
            float qf[8];
            unpack_magic<KB>(lo[u][k], hi[u][k], bits, qf);
#pragma unroll
            for (int j = 0; j < 8; ++j) x[k][j] = __fadd_rn(x[k][j], __fmaf_rn(un[u], qf[j], mi[u]));
          }
        }
      }
    }
    return;
  }
  constexpr int kB = SliceCfg<GPL>::kPeerBatch;
  for (int i0 = 0; i0 < cnt; i0 += kB) {
    SliceWords<GPL> w[kB];
#pragma unroll
    for (int u = 0; u < kB; ++u) {
      const int i = i0 + u;
      if (i < cnt) {
        const int q = (ss.skip >= 0 && i >= ss.skip) ? i + 1 : i;
        slice_fetch<KB, GPL>(ss.base + (size_t)q * ss.stride, meta_off, pay_off, lg, bits, w[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < kB; ++u)
      if (i0 + u < cnt) slice_decode<KB, GPL, true>(w[u], bits, x);
  }
}

// ======================================================================================
// full items, values already in registers (x = raw loaded values, not yet prescaled)
// ======================================================================================
// TO: element type of the self-decoded output (SELF only)
template <typename TO, int KB, int GPL, bool SELF, bool VEC, typename DST>
__device__ __forceinline__ void full_send_x(float (&x)[GPL][8], const WarpItem& it, float prescale, const RngKey& rng,
                                            const DST& ds, TO* __restrict__ self_out) {
  const int bits = KB ? KB : item_bits(it);
  const uint32_t lg = item_lpb_log2(it);
  slice_scale<GPL>(x, prescale);
  BucketMeta m[GPL];
  float inv[GPL];
  slice_meta<GPL>(x, lg, bits, m, inv);
  slice_store_meta<GPL>(m, lg, ds, it.meta_off);
  slice_encode<TO, KB, GPL, SELF, VEC>(x, m, inv, bits, rng, it.elem_off, ds, it.pay_off, self_out);
}

template <typename T, int KB, int GPL, bool VEC, typename DST>
__device__ __forceinline__ void full_reduce_x(float (&x)[GPL][8], T* __restrict__ blk, const WarpItem& it,
                                              float prescale, const RngKey& rng, const SrcSet& ss, const DST& ds) {
  const int bits = KB ? KB : item_bits(it);
  const uint32_t lg = item_lpb_log2(it);
  slice_scale<GPL>(x, prescale);
  slice_accumulate<KB, GPL>(ss, it.meta_off, it.pay_off, lg, bits, x);
  BucketMeta m[GPL];
  float inv[GPL];
  slice_meta<GPL>(x, lg, bits, m, inv);
  slice_store_meta<GPL>(m, lg, ds, it.meta_off);
  slice_encode<T, KB, GPL, true, VEC>(x, m, inv, bits, rng, it.elem_off, ds, it.pay_off, blk);
}

// out = decode(already fetched words of ONE source)
template <typename TO, int KB, int GPL, bool VEC>
__device__ __forceinline__ void full_recv_w(const SliceWords<GPL>& w, const WarpItem& it, TO* __restrict__ out) {
  const int bits = KB ? KB : item_bits(it);
  float x[GPL][8];
  slice_decode<KB, GPL, false>(w, bits, x);
  slice_store<TO, GPL, VEC>(out, x);
}

// out = sum of all sources, slot order (one-shot phase 2)
template <typename TO, int KB, int GPL, bool VEC>
__device__ __forceinline__ void full_recv_sum(const SrcSet& ss, const WarpItem& it, TO* __restrict__ out) {
  const int bits = KB ? KB : item_bits(it);
  const uint32_t lg = item_lpb_log2(it);
  float x[GPL][8];
#pragma unroll
  for (int k = 0; k < GPL; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) x[k][j] = 0.f;
  slice_accumulate<KB, GPL>(ss, it.meta_off, it.pay_off, lg, bits, x);
  slice_store<TO, GPL, VEC>(out, x);
}

// ---- two items at once ------------------------------------------------------------------
// With 16 warps per SM the dependent chains of one item (min/max tree -> redux -> reciprocal ->
// encode -> pack) leave the schedulers idle; two independent items in ONE basic block give the
// compiler twice the instruction-level parallelism. Only the common case qualifies: both slices
// are a single bucket, deterministic rounding, finite values. Returns false (nothing done) if not.
template <int GPL>
__device__ __forceinline__ void slice_meta_single(const float (&x)[GPL][8], int bits, BucketMeta& m, float& inv) {
  float mn = CGX_INF_POS, mx = CGX_INF_NEG;
#pragma unroll
  for (int k = 0; k < GPL; ++k) minmax8(x[k], mn, mx);
  warp_minmax(mn, mx);
  m = make_meta(mn, mx, bits);
  inv = inv_unit(m.unit);
}

template <int KB, int GPL, typename DST>
__device__ __forceinline__ bool full_send_pair(float (&xa)[GPL][8], float (&xb)[GPL][8], const WarpItem& ita,
                                               const WarpItem& itb, float prescale, const RngKey& rng,
                                               const DST& dsa, const DST& dsb) {
  if (rng.enabled || !slice_single_bucket<GPL>(item_lpb_log2(ita)) || !slice_single_bucket<GPL>(item_lpb_log2(itb)))
    return false;
  const int bits_a = KB ? KB : item_bits(ita), bits_b = KB ? KB : item_bits(itb);
  slice_scale<GPL>(xa, prescale);
  slice_scale<GPL>(xb, prescale);
  BucketMeta ma, mb;
  float ia, ib;
  slice_meta_single<GPL>(xa, bits_a, ma, ia);
  slice_meta_single<GPL>(xb, bits_b, mb, ib);
  if (lane_id() == 0) {
    dst_st_v2(dsa, ita.meta_off, __float_as_uint(ma.unit), __float_as_uint(ma.min));
    dst_st_v2(dsb, itb.meta_off, __float_as_uint(mb.unit), __float_as_uint(mb.min));
  }
  const bool finite = __all_sync(kAll, fabsf(ma.unit) < CGX_INF_POS && fabsf(mb.unit) < CGX_INF_POS);
  BucketMeta mav[GPL], mbv[GPL];
  float iav[GPL], ibv[GPL];
#pragma unroll
  for (int k = 0; k < GPL; ++k) {
    mav[k] = ma;
    mbv[k] = mb;
    iav[k] = ia;
    ibv[k] = ib;
  }
  if (finite) {
    // interleave by rows so that both items' chains are in flight together
    const float maxa = (float)max_level(bits_a), maxb = (float)max_level(bits_b);
    uint32_t loa[GPL], hia[GPL], lob[GPL], hib[GPL];
#pragma unroll
    for (int k = 0; k < GPL; ++k) {
      float ua[8], ub[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        ua[j] = level_magic<false>(xa[k][j], ma.min, ia, 0.5f, maxa);
        ub[j] = level_magic<false>(xb[k][j], mb.min, ib, 0.5f, maxb);
      }
      pack_magic<KB>(ua, bits_a, loa[k], hia[k]);
      pack_magic<KB>(ub, bits_b, lob[k], hib[k]);
    }
    store_words<KB, GPL>(dsa, ita.pay_off, bits_a, loa, hia);
    store_words<KB, GPL>(dsb, itb.pay_off, bits_b, lob, hib);
  } else {
    slice_encode_mode<float, KB, GPL, false, true, 1>(xa, mav, iav, bits_a, rng, ita.elem_off, dsa, ita.pay_off,
                                                      (float*)nullptr);
    slice_encode_mode<float, KB, GPL, false, true, 1>(xb, mbv, ibv, bits_b, rng, itb.elem_off, dsb, itb.pay_off,
                                                      (float*)nullptr);
  }
  return true;
}

// decode two already fetched items (branch free: the two chains interleave)
template <typename TO, int KB, int GPL>
__device__ __forceinline__ void full_recv_pair(const SliceWords<GPL>& wa, const SliceWords<GPL>& wb,
                                               const WarpItem& ita, const WarpItem& itb, TO* __restrict__ oa,
                                               TO* __restrict__ ob) {
  const int bits_a = KB ? KB : item_bits(ita), bits_b = KB ? KB : item_bits(itb);
  float xa[GPL][8], xb[GPL][8];
  slice_decode<KB, GPL, false>(wa, bits_a, xa);
  slice_decode<KB, GPL, false>(wb, bits_b, xb);
  slice_store<TO, GPL, true>(oa, xa);
  slice_store<TO, GPL, true>(ob, xb);
}

// ---- the same for slices whose gradients are not vector aligned: out of line, scalar access ----
template <typename TS, typename TO, int KB, int GPL, bool SELF, typename DST>
__device__ __noinline__ void full_send_unaligned(const TS* __restrict__ src, const WarpItem it, float prescale,
                                                 const RngKey rng, const DST ds, TO* __restrict__ self_out) {
  float x[GPL][8];
  slice_load_scalar<TS, GPL>(src, x);
  full_send_x<TO, KB, GPL, SELF, false>(x, it, prescale, rng, ds, self_out);
}
template <typename T, int KB, int GPL, typename DST>
__device__ __noinline__ void full_reduce_unaligned(T* __restrict__ blk, const WarpItem it, float prescale,
                                                   const RngKey rng, const SrcSet ss, const DST ds) {
  float x[GPL][8];
  slice_load_scalar<T, GPL>(blk, x);
  full_reduce_x<T, KB, GPL, false>(x, blk, it, prescale, rng, ss, ds);
}
template <typename TO, int KB, int GPL>
__device__ __noinline__ void full_recv_unaligned(const SrcSet ss, const WarpItem it, TO* __restrict__ out) {
  if (ss.n == 1) {
    SliceWords<GPL> w;
    slice_fetch<KB, GPL>(ss.base, it.meta_off, it.pay_off, item_lpb_log2(it), KB ? KB : item_bits(it), w);
    full_recv_w<TO, KB, GPL, false>(w, it, out);
  } else {
    full_recv_sum<TO, KB, GPL, false>(ss, it, out);
  }
}

// ======================================================================================
// generic bucket items (cold): ONE bucket of n <= kMaxBlockElems elements, any alignment,
// any bit width. Two passes (min/max, then encode); lane l handles groups l, l+32, ...
// ======================================================================================
// ROUND: the products are rounded to TS as well, x = TS(x * prescale) (scale_round)
template <typename TS, bool ROUND = false>
__device__ __forceinline__ void bucket_load_group(const TS* __restrict__ src, uint32_t g, uint32_t n, float prescale,
                                                  float (&x)[8], int& nv) {
  nv = (int)min(8u, n - g * 8u);
  load8_scalar<TS>(src + g * 8u, nv, x);
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] = ROUND ? scale_round<TS>(x[j], prescale) : __fmul_rn(x[j], prescale);
}

__device__ __forceinline__ void bucket_add_sources(const SrcSet& ss, const WarpItem& it, uint32_t g, int bits,
                                                   float (&x)[8]) {
  for (int q = 0; q < ss.n; ++q) {
    if (q == ss.skip) continue;
    const uint8_t* rec = ss.base + (size_t)q * ss.stride;
    uint32_t lo, hi;
    load_word<0>(rec + it.pay_off, g, bits, lo, hi);
    const uint2 mv = ld_sys_v2(rec + it.meta_off);
    float qf[8];
    unpack_magic<0>(lo, hi, bits, qf);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      x[j] = __fadd_rn(x[j], __fmaf_rn(__uint_as_float(mv.x), qf[j], __uint_as_float(mv.y)));
  }
}

// phase A / phase B / quantize of a generic bucket. `ss.n == 0`: nothing to add (send);
// self_out != nullptr: write the self-decoded values there; ROUND: as bucket_load_group
template <typename TS, typename TO, typename DST, bool ROUND>
__device__ __forceinline__ void bucket_quantize_body(const TS* __restrict__ src, const WarpItem& it, float prescale,
                                                     const RngKey& rng, const SrcSet& ss, const DST& ds,
                                                     TO* __restrict__ self_out) {
  const uint32_t n = item_n(it);
  const int bits = item_bits(it);
  const uint32_t ng = div_up(n, 8u);
  float mn = CGX_INF_POS, mx = CGX_INF_NEG;
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
    int nv;
    bucket_load_group<TS, ROUND>(src, g, n, prescale, x, nv);
    if (ss.n > 0) bucket_add_sources(ss, it, g, bits, x);
    minmax8_pred(x, nv, mn, mx);
  }
  warp_minmax(mn, mx);
  const BucketMeta m = make_meta(mn, mx, bits);
  const float inv = inv_unit(m.unit);
  const float maxlvl = (float)max_level(bits);
  // generic items always use the unicast mappings (sub-word stores have no multimem form)
  const DST du = unicast_of(ds);
  if (lane_id() == 0) dst_st_v2(du, it.meta_off, __float_as_uint(m.unit), __float_as_uint(m.min));
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
    int nv;
    bucket_load_group<TS, ROUND>(src, g, n, prescale, x, nv);
    if (ss.n > 0) bucket_add_sources(ss, it, g, bits, x);
    float r[8];
    if (rng.enabled) {
      rounding8(rng, it.elem_off + g * 8u, r);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = 0.5f;
    }
    float u[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) u[j] = (j < nv) ? level_magic<true>(x[j], m.min, inv, r[j], maxlvl) : CGX_MAGIC;
    uint32_t lo, hi;
    pack_magic<0>(u, bits, lo, hi);
    // byte-granular store (a bucket's payload may start at any byte offset)
    {
      const uint64_t w = (uint64_t)lo | ((uint64_t)hi << 32);
      const uint32_t o = it.pay_off + g * (uint32_t)bits;
      for (int t = 0; t < bits; ++t) dst_st_u8(du, o + t, (uint32_t)(w >> (8 * t)) & 0xFFu);
    }
    if (self_out != nullptr) {
      float dec[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) dec[j] = __fmaf_rn(m.unit, __fsub_rn(u[j], CGX_MAGIC), m.min);
      store8_scalar<TO>(self_out + g * 8u, nv, dec);
    }
  }
}
template <typename TS, typename TO, typename DST>
__device__ __noinline__ void bucket_quantize(const TS* __restrict__ src, const WarpItem it, float prescale,
                                             const RngKey rng, const SrcSet ss, const DST ds,
                                             TO* __restrict__ self_out) {
  bucket_quantize_body<TS, TO, DST, false>(src, it, prescale, rng, ss, ds, self_out);
}
// send of the generic bucket of TS(src * scale) (scale_round)
template <typename TS, typename DST>
__device__ __noinline__ void bucket_quantize_rounded(const TS* __restrict__ src, const WarpItem it, float scale,
                                                     const RngKey rng, const DST ds) {
  bucket_quantize_body<TS, TS, DST, true>(src, it, scale, rng, SrcSet{nullptr, 0u, 0, -1}, ds, (TS*)nullptr);
}

// decode one source (ss.n == 1) or the sum of all sources into `out`
template <typename TO>
__device__ __noinline__ void bucket_recv(const SrcSet ss, const WarpItem it, TO* __restrict__ out) {
  const uint32_t n = item_n(it);
  const int bits = item_bits(it);
  const uint32_t ng = div_up(n, 8u);
  SrcSet s2 = ss;
  s2.skip = -1;
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = 0.f;
    bucket_add_sources(s2, it, g, bits, x);  // 0 + d == d exactly
    store8_scalar<TO>(out + g * 8u, (int)min(8u, n - g * 8u), x);
  }
}

// ======================================================================================
// raw (uncompressed) items: n <= 512 elements travelling as T
// ======================================================================================
// 8 values -> 8 T on the wire (16 B-aligned records): 2 x 16 B for fp32, 1 x 16 B otherwise
template <typename T, typename DST>
__device__ __forceinline__ void raw_wire_store(const DST& ds, uint32_t off, const float (&v)[8]) {
  if (sizeof(T) == 4) {
    dst_st_v4(ds, off, pack16<T>(v));
    dst_st_v4(ds, off + 16u, pack16<T>(v + 4));
  } else {
    dst_st_v4(ds, off, pack16<T>(v));
  }
}
template <typename T>
__device__ __forceinline__ void raw_wire_load(const uint8_t* p, float (&v)[8]) {
  if (sizeof(T) == 4) {
    unpack16<T>(ld_sys_v4(p), v);
    unpack16<T>(ld_sys_v4(p + 16), v + 4);
  } else {
    unpack16<T>(ld_sys_v4(p), v);
  }
}

// Full raw item (512 elements, vector-aligned gradients); x = the item's raw loaded values (MODE 0/1)
//   MODE 0: push (phase A / one-shot 1): dst <- T(x * prescale)
//   MODE 1: reduce (phase B): x * prescale + sum(sources) -> own, dst
//   MODE 2: receive: out <- source (ss.n == 1) or sum of all sources
//   MODE 3: reduce-scatter: x * prescale + sum(sources) -> blk (the output shard) only
// (x may have more than 2 rows -- the prefetch buffer of a 1024 slice -- only rows 0 and 1 are used)
template <typename T, int MODE, int ROWS, typename DST>
__device__ __forceinline__ void raw_full_x(float (&x)[ROWS][8], T* __restrict__ blk, const WarpItem& it,
                                           float prescale, const SrcSet& ss, const DST& ds) {
#pragma unroll
  for (int k = 0; k < 2; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) x[k][j] = MODE == 2 ? 0.f : __fmul_rn(x[k][j], prescale);
  if (MODE != 0) {
    for (int q = 0; q < ss.n; ++q) {
      if (q == ss.skip) continue;
      const uint8_t* rec = ss.base + (size_t)q * ss.stride + it.meta_off;
      float v[2][8];
#pragma unroll
      for (int k = 0; k < 2; ++k) raw_wire_load<T>(rec + (lane_id() * 2u + (uint32_t)k) * 8u * sizeof(T), v[k]);
#pragma unroll
      for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) x[k][j] = __fadd_rn(x[k][j], v[k][j]);
    }
  }
  if (MODE == 0 || MODE == 1) {
#pragma unroll
    for (int k = 0; k < 2; ++k)
      raw_wire_store<T>(ds, it.meta_off + (lane_id() * 2u + (uint32_t)k) * 8u * (uint32_t)sizeof(T), x[k]);
  }
  if (MODE != 0) {
    T* o = blk + lane_id() * 16u;
#pragma unroll
    for (int k = 0; k < 2; ++k) store8_vec<T>(o + k * 8, x[k]);
  }
}
// rows 0..1 of a (possibly larger) register buffer <- the 512 elements of a raw item
template <typename T, int ROWS>
__device__ __forceinline__ void raw_load_vec(const T* __restrict__ src, float (&x)[ROWS][8]) {
  const T* p = src + lane_id() * 16u;
#pragma unroll
  for (int k = 0; k < 2; ++k) load8_vec<T>(p + k * 8, x[k]);
}

// In-switch reduction of a full raw item (NVLS): every rank staged T(src * prescale) at the same
// heap offset; the owner pulls the sum with multimem.ld_reduce and multicasts it back in place.
template <typename T>
__device__ __forceinline__ void raw_full_mc_reduce(T* __restrict__ blk, const WarpItem& it, uint8_t* mc_slot) {
  constexpr uint32_t kVecs = 512u * sizeof(T) / 16u / 32u;  // 16 B vectors per lane: 4 (fp32) or 2
  uint4 v[kVecs];
#pragma unroll
  for (uint32_t i = 0; i < kVecs; ++i) v[i] = mc_ld_reduce_v4<T>(mc_slot + it.meta_off + (i * 32u + lane_id()) * 16u);
  const bool vec = (reinterpret_cast<uintptr_t>(blk) & 15u) == 0;
#pragma unroll
  for (uint32_t i = 0; i < kVecs; ++i) {
    const uint32_t byte = (i * 32u + lane_id()) * 16u;
    mc_st_v4(mc_slot + it.meta_off + byte, v[i]);
    T* o = blk + byte / sizeof(T);
    if (vec) {
      *reinterpret_cast<uint4*>(o) = v[i];
    } else {
      const T* pe = reinterpret_cast<const T*>(&v[i]);
#pragma unroll
      for (uint32_t j = 0; j < 16u / sizeof(T); ++j) o[j] = pe[j];
    }
  }
}

// raw tail (< 512 elements) or a full raw item with unaligned gradients: element-wise, cold.
// mode as in raw_full_x.
template <typename T, typename DST>
__device__ __noinline__ void raw_generic(T* __restrict__ blk, const WarpItem it, float prescale, const SrcSet ss,
                                         const DST ds, int mode) {
  const uint32_t n = item_n(it);
  const DST du = unicast_of(ds);
  for (uint32_t i = lane_id(); i < n; i += 32) {
    float x = mode == 2 ? 0.f : __fmul_rn(DT<T>::to_float(blk[i]), prescale);
    if (mode != 0) {
      for (int q = 0; q < ss.n; ++q) {
        if (q == ss.skip) continue;
        const T* rec = reinterpret_cast<const T*>(ss.base + (size_t)q * ss.stride + it.meta_off);
        T v;
        if (sizeof(T) == 4) {
          const uint32_t b = ld_sys_u32(rec + i);
          v = *reinterpret_cast<const T*>(&b);
        } else {
          const uint16_t b = (uint16_t)ld_sys_u16(rec + i);
          v = *reinterpret_cast<const T*>(&b);
        }
        x = __fadd_rn(x, DT<T>::to_float(v));
      }
    }
    const T t = DT<T>::from_float(x);
    if (mode != 2) {
      const uint32_t o = it.meta_off + i * (uint32_t)sizeof(T);
      if (sizeof(T) == 4)
        dst_st_u32(du, o, *reinterpret_cast<const uint32_t*>(&t));
      else
        dst_st_u16(du, o, *reinterpret_cast<const uint16_t*>(&t));
    }
    if (mode != 0) blk[i] = t;
  }
}

// ======================================================================================
// reduce-scatter (rs_kernel phase B): my values * prescale + the decoded copies of the W-1
// sources, in slot order, stored as T to the output shard. Nothing is requantized or published.
// `src` and `out` are either disjoint or the same address (output aliasing my input chunk):
// every lane reads an element before it writes it, so they carry no __restrict__.
// ======================================================================================
template <typename T, int KB, int GPL, bool VEC>
__device__ __forceinline__ void full_rs_x(float (&x)[GPL][8], const WarpItem& it, float prescale, const SrcSet& ss,
                                          T* out) {
  const int bits = KB ? KB : item_bits(it);
  slice_scale<GPL>(x, prescale);
  slice_accumulate<KB, GPL>(ss, it.meta_off, it.pay_off, item_lpb_log2(it), bits, x);
  slice_store<T, GPL, VEC>(out, x);
}
template <typename T, int KB, int GPL>
__device__ __noinline__ void full_rs_unaligned(const T* src, const WarpItem it, float prescale, const SrcSet ss,
                                               T* out) {
  float x[GPL][8];
  slice_load_scalar<T, GPL>(src, x);
  full_rs_x<T, KB, GPL, false>(x, it, prescale, ss, out);
}

template <typename T>
__device__ __noinline__ void bucket_rs(const T* src, const WarpItem it, float prescale, const SrcSet ss, T* out) {
  const uint32_t n = item_n(it);
  const int bits = item_bits(it);
  const uint32_t ng = div_up(n, 8u);
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
    int nv;
    bucket_load_group<T>(src, g, n, prescale, x, nv);
    bucket_add_sources(ss, it, g, bits, x);
    store8_scalar<T>(out + g * 8u, nv, x);
  }
}

// raw tail, or a full raw item whose input or output is not vector aligned: element-wise
template <typename T>
__device__ __noinline__ void raw_rs_generic(const T* src, const WarpItem it, float prescale, const SrcSet ss,
                                            T* out) {
  const uint32_t n = item_n(it);
  for (uint32_t i = lane_id(); i < n; i += 32) {
    float x = __fmul_rn(DT<T>::to_float(src[i]), prescale);
    for (int q = 0; q < ss.n; ++q) {
      if (q == ss.skip) continue;
      const T* rec = reinterpret_cast<const T*>(ss.base + (size_t)q * ss.stride + it.meta_off);
      T v;
      if (sizeof(T) == 4) {
        const uint32_t b = ld_sys_u32(rec + i);
        v = *reinterpret_cast<const T*>(&b);
      } else {
        const uint16_t b = (uint16_t)ld_sys_u16(rec + i);
        v = *reinterpret_cast<const T*>(&b);
      }
      x = __fadd_rn(x, DT<T>::to_float(v));
    }
    out[i] = DT<T>::from_float(x);
  }
}

// ======================================================================================
// all-gather (ag_kernel publish): a raw item travels as T to every peer and the same T lands in my
// output. The compressed kinds use *_send / bucket_quantize with their self-decoded output.
// ======================================================================================
// rows 0..1 of x (a full raw item after raw_full_x MODE 0) -> the 512 elements at `dst`
template <typename T, int ROWS>
__device__ __forceinline__ void raw_store_vec(T* __restrict__ dst, const float (&x)[ROWS][8]) {
  T* p = dst + lane_id() * 16u;
#pragma unroll
  for (int k = 0; k < 2; ++k) store8_vec<T>(p + k * 8, x[k]);
}

// raw tail, or a full raw item whose input or output is not vector aligned: element-wise.
// `src` and `out` are disjoint or the same address (every lane reads an element before it writes it).
template <typename T, typename DST>
__device__ __noinline__ void raw_ag_generic(const T* src, const WarpItem it, float prescale, const DST ds, T* out) {
  const uint32_t n = item_n(it);
  const DST du = unicast_of(ds);
  for (uint32_t i = lane_id(); i < n; i += 32) {
    const T t = DT<T>::from_float(__fmul_rn(DT<T>::to_float(src[i]), prescale));
    const uint32_t o = it.meta_off + i * (uint32_t)sizeof(T);
    if (sizeof(T) == 4)
      dst_st_u32(du, o, *reinterpret_cast<const uint32_t*>(&t));
    else
      dst_st_u16(du, o, *reinterpret_cast<const uint16_t*>(&t));
    out[i] = t;
  }
}

// all-gather decode of a raw item from ONE source (ss.n == 1): the record's T values unchanged, so a
// peer's copy has the owner's bits (raw_full_x / raw_generic receive as 0 + v, which turns -0 into +0)
template <typename T>
__device__ __noinline__ void raw_ag_recv(const SrcSet ss, const WarpItem it, T* __restrict__ out) {
  const uint8_t* rec = ss.base + it.meta_off;
  if (item_kind(it) == kItemRaw && group_aligned<T>(out)) {
    float v[2][8];
#pragma unroll
    for (int k = 0; k < 2; ++k) raw_wire_load<T>(rec + (lane_id() * 2u + (uint32_t)k) * 8u * sizeof(T), v[k]);
    raw_store_vec<T, 2>(out, v);
    return;
  }
  const uint32_t n = item_n(it);
  for (uint32_t i = lane_id(); i < n; i += 32) {
    if (sizeof(T) == 4) {
      const uint32_t b = ld_sys_u32(rec + i * 4u);
      out[i] = *reinterpret_cast<const T*>(&b);
    } else {
      const uint16_t b = (uint16_t)ld_sys_u16(rec + i * 2u);
      out[i] = *reinterpret_cast<const T*>(&b);
    }
  }
}

// ======================================================================================
// FP8 codecs of the compressed all-to-all (quant_math.h, CODEC = kE4M3 / kE5M2 and the Pow2 twins): 8-bit records
// whose meta is {unit, +0} and whose byte j of a group is element j's FP8 code. Same slices, same
// min/max reductions and the same 8-bit word loads and stores as max-min; only the element
// arithmetic differs: one FMUL + half a cvt.satfinite per element to encode, half a cvt.f16x2 +
// one F2F + one FMUL to decode. The SR codecs (fp8_sr) add one Philox call per group of 8 and a few
// integer operations per element (fp8_sr_snap); every encoder takes the key and the item's element
// index, which the round-to-nearest codecs ignore.
// ======================================================================================
// per-row NaN-propagating min / max of the bucket each row of the slice belongs to (slice_meta's
// reductions)
template <int GPL>
__device__ __forceinline__ void slice_minmax(const float (&x)[GPL][8], uint32_t lg, float (&mn)[GPL],
                                             float (&mx)[GPL]) {
#pragma unroll
  for (int k = 0; k < GPL; ++k) {
    mn[k] = CGX_INF_POS;
    mx[k] = CGX_INF_NEG;
    minmax8(x[k], mn[k], mx[k]);
  }
  if (lg == 0) return;  // 8-element buckets: every row is its own bucket
  float a = mn[0], b = mx[0];
#pragma unroll
  for (int k = 1; k < GPL; ++k) {
    a = nan_min(a, mn[k]);
    b = nan_max(b, mx[k]);
  }
  if (slice_single_bucket<GPL>(lg))
    warp_minmax(a, b);
  else
    subwarp_minmax(a, b, lg - 1u);  // (512-slices only) a bucket = all rows of 2^(lg-1) adjacent lanes
#pragma unroll
  for (int k = 0; k < GPL; ++k) {
    mn[k] = a;
    mx[k] = b;
  }
}

// 8 values of one group -> their codes, element j in byte j of (lo, hi). An SR codec rounds element j
// with half j of the Philox word of the group's first element `first` (quantize_block_fp8's bits).
template <int CODEC>
__device__ __forceinline__ void fp8_encode8(const float (&x)[8], float inv, const RngKey& rng, uint32_t first,
                                            uint32_t& lo, uint32_t& hi) {
  uint32_t p0, p1, p2, p3;
  if constexpr (fp8_sr(CODEC)) {
    const Philox4 a = rounding_word(rng, first);
    p0 = fp8x2_encode_sr(x[0], x[1], inv, CODEC, a.v[0], a.v[0] >> 16);
    p1 = fp8x2_encode_sr(x[2], x[3], inv, CODEC, a.v[1], a.v[1] >> 16);
    p2 = fp8x2_encode_sr(x[4], x[5], inv, CODEC, a.v[2], a.v[2] >> 16);
    p3 = fp8x2_encode_sr(x[6], x[7], inv, CODEC, a.v[3], a.v[3] >> 16);
  } else {
    p0 = fp8x2_encode(x[0], x[1], inv, CODEC), p1 = fp8x2_encode(x[2], x[3], inv, CODEC);
    p2 = fp8x2_encode(x[4], x[5], inv, CODEC), p3 = fp8x2_encode(x[6], x[7], inv, CODEC);
  }
  lo = __byte_perm(p0, p1, 0x5410);
  hi = __byte_perm(p2, p3, 0x5410);
}
template <int CODEC>
__device__ __forceinline__ void fp8_decode8(uint32_t lo, uint32_t hi, float unit, float (&x)[8]) {
  fp8x2_decode(lo, unit, CODEC, x[0], x[1]);
  fp8x2_decode(lo >> 16, unit, CODEC, x[2], x[3]);
  fp8x2_decode(hi, unit, CODEC, x[4], x[5]);
  fp8x2_decode(hi >> 16, unit, CODEC, x[6], x[7]);
}

// full item, values already in registers: meta + codes to the destination; the codes stay in
// (lo, hi) and the units in m for a caller that decodes them itself
template <int CODEC, int GPL, typename DST>
__device__ __forceinline__ void full_send_fp8_codes(const float (&x)[GPL][8], const WarpItem& it, const RngKey& rng,
                                                    const DST& ds, BucketMeta (&m)[GPL], uint32_t (&lo)[GPL],
                                                    uint32_t (&hi)[GPL]) {
  const uint32_t lg = item_lpb_log2(it);
  float mn[GPL], mx[GPL];
  slice_minmax<GPL>(x, lg, mn, mx);
#pragma unroll
  for (int k = 0; k < GPL; ++k) {
    m[k] = fp8_meta(mn[k], mx[k], CODEC);
    fp8_encode8<CODEC>(x[k], fp8_inv_unit(m[k].unit, CODEC), rng, it.elem_off + lane_group<GPL>(k) * 8u, lo[k], hi[k]);
  }
  slice_store_meta<GPL>(m, lg, ds, it.meta_off);
  store_words<8, GPL>(ds, it.pay_off, 8, lo, hi);
}
template <int CODEC, int GPL, typename DST>
__device__ __forceinline__ void full_send_fp8_x(const float (&x)[GPL][8], const WarpItem& it, const RngKey& rng,
                                                const DST& ds) {
  BucketMeta m[GPL];
  uint32_t lo[GPL], hi[GPL];
  full_send_fp8_codes<CODEC, GPL>(x, it, rng, ds, m, lo, hi);
}
template <typename TS, int CODEC, int GPL, typename DST>
__device__ __noinline__ void full_send_fp8_unaligned(const TS* __restrict__ src, const WarpItem it, const RngKey rng,
                                                     const DST ds) {
  float x[GPL][8];
  slice_load_scalar<TS, GPL>(src, x);
  full_send_fp8_x<CODEC, GPL>(x, it, rng, ds);
}

// out = decode(already fetched words of ONE source)
template <typename TO, int CODEC, int GPL, bool VEC>
__device__ __forceinline__ void full_recv_fp8_w(const SliceWords<GPL>& w, TO* __restrict__ out) {
  float x[GPL][8];
#pragma unroll
  for (int k = 0; k < GPL; ++k) fp8_decode8<CODEC>(w.lo[k], w.hi[k], w.pm[k].unit, x[k]);
  slice_store<TO, GPL, VEC>(out, x);
}
template <typename TO, int CODEC, int GPL>
__device__ __noinline__ void full_recv_fp8_unaligned(const uint8_t* rec, const WarpItem it, TO* __restrict__ out) {
  SliceWords<GPL> w;
  slice_fetch<8, GPL>(rec, it.meta_off, it.pay_off, item_lpb_log2(it), 8, w);
  full_recv_fp8_w<TO, CODEC, GPL, false>(w, out);
}

// generic bucket item (cold): ONE bucket of n <= kMaxBlockElems elements, any alignment; the codes
// of the last group's missing elements are 0, as on the host
// of the values src * prescale; self_out != nullptr: also the values decoded from the codes there;
// ROUND: as bucket_load_group
template <typename TS, typename TO, int CODEC, typename DST, bool ROUND = false>
__device__ __forceinline__ void bucket_fp8_body(const TS* __restrict__ src, const WarpItem& it, float prescale,
                                                const RngKey& rng, const DST& ds, TO* __restrict__ self_out) {
  const uint32_t n = item_n(it);
  const uint32_t ng = div_up(n, 8u);
  float mn = CGX_INF_POS, mx = CGX_INF_NEG;
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
    int nv;
    bucket_load_group<TS, ROUND>(src, g, n, prescale, x, nv);
    minmax8_pred(x, nv, mn, mx);
  }
  warp_minmax(mn, mx);
  const BucketMeta m = fp8_meta(mn, mx, CODEC);
  const float inv = fp8_inv_unit(m.unit, CODEC);
  const DST du = unicast_of(ds);
  if (lane_id() == 0) dst_st_v2(du, it.meta_off, __float_as_uint(m.unit), __float_as_uint(m.min));
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
    int nv;
    bucket_load_group<TS, ROUND>(src, g, n, prescale, x, nv);
    uint32_t lo, hi;
    fp8_encode8<CODEC>(x, inv, rng, it.elem_off + g * 8u, lo, hi);
    const uint64_t w = ((uint64_t)hi << 32 | lo) & (nv >= 8 ? ~0ull : (1ull << (8 * nv)) - 1ull);
    const uint32_t o = it.pay_off + g * 8u;
    for (int t = 0; t < 8; ++t) dst_st_u8(du, o + t, (uint32_t)(w >> (8 * t)) & 0xFFu);
    if (self_out != nullptr) {
      float dec[8];
      fp8_decode8<CODEC>(lo, hi, m.unit, dec);
      store8_scalar<TO>(self_out + g * 8u, nv, dec);
    }
  }
}
template <typename TS, int CODEC, typename DST>
__device__ __noinline__ void bucket_quantize_fp8(const TS* __restrict__ src, const WarpItem it, const RngKey rng,
                                                 const DST ds) {
  bucket_fp8_body<TS, float, CODEC>(src, it, 1.0f, rng, ds, (float*)nullptr);
}
// the same for the bucket of TS(src * scale) (scale_round)
template <typename TS, int CODEC, typename DST>
__device__ __noinline__ void bucket_quantize_fp8_rounded(const TS* __restrict__ src, const WarpItem it, float scale,
                                                         const RngKey rng, const DST ds) {
  bucket_fp8_body<TS, float, CODEC, DST, true>(src, it, scale, rng, ds, (float*)nullptr);
}

template <typename TO, int CODEC>
__device__ __noinline__ void bucket_recv_fp8(const uint8_t* rec, const WarpItem it, TO* __restrict__ out) {
  const uint32_t n = item_n(it);
  const uint32_t ng = div_up(n, 8u);
  const float unit = __uint_as_float(ld_sys_v2(rec + it.meta_off).x);
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    uint32_t lo, hi;
    load_word<0>(rec + it.pay_off, g, 8, lo, hi);
    float x[8];
    fp8_decode8<CODEC>(lo, hi, unit, x);
    store8_scalar<TO>(out + g * 8u, (int)min(8u, n - g * 8u), x);
  }
}

// ---- FP8 codes handed to the caller undecoded (the all-to-all's and all-gather's codes output) -----
// Inside an item the codes of an FP8 record are in element order (full items: group g at pay_off +
// 8g; bucket items: one bucket, byte i at pay_off + i), so element e of the item is codes[e] and the
// unit of its bucket b is scales[b]: unpacking is a copy.
//
// The destination that lets the FP8 encoders write an item straight to (codes, scales): a meta store
// (dst_st_v2: only metas use it in the FP8 encoders) keeps the unit, payload stores land at
// codes + (off - pay_off), and the bytes past the item's n elements (a bucket's padding) are dropped.
struct CodesDst {
  uint8_t* codes;
  float* scales;
  uint32_t meta_off, pay_off, n;
};
__device__ __forceinline__ CodesDst unicast_of(const CodesDst& ds) { return ds; }
__device__ __forceinline__ void dst_st_v2(const CodesDst& ds, uint32_t off, uint32_t a, uint32_t) {
  ds.scales[(off - ds.meta_off) >> 3] = __uint_as_float(a);
}
__device__ __forceinline__ void dst_st_u8(const CodesDst& ds, uint32_t off, uint32_t v) {
  const uint32_t o = off - ds.pay_off;
  if (o < ds.n) st_u8(ds.codes + o, v);
}
// 16 payload bytes of a full item (never past n: full items are whole slices)
__device__ __forceinline__ void dst_st_v4(const CodesDst& ds, uint32_t off, const uint4& v) {
  uint8_t* d = ds.codes + (off - ds.pay_off);
  if ((reinterpret_cast<uintptr_t>(d) & 15u) == 0) {
    st_v4(d, v);
    return;
  }
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int t = 0; t < 16; ++t) st_u8(d + t, (w[t >> 2] >> (8 * (t & 3))) & 0xFFu);
}

// The all-gather owner's codes output: every store of the FP8 encoder goes to the peers' slots and
// to the owner's (codes, scales), so the owner keeps exactly the bytes it published.
template <typename D>
struct TeeDst {
  D peers;
  CodesDst own;
};
template <typename D>
__device__ __forceinline__ TeeDst<D> unicast_of(const TeeDst<D>& ds) {
  return TeeDst<D>{unicast_of(ds.peers), ds.own};
}
template <typename D>
__device__ __forceinline__ void dst_st_v2(const TeeDst<D>& ds, uint32_t off, uint32_t a, uint32_t b) {
  dst_st_v2(ds.peers, off, a, b);
  dst_st_v2(ds.own, off, a, b);
}
template <typename D>
__device__ __forceinline__ void dst_st_u8(const TeeDst<D>& ds, uint32_t off, uint32_t v) {
  dst_st_u8(ds.peers, off, v);
  dst_st_u8(ds.own, off, v);
}
template <typename D>
__device__ __forceinline__ void dst_st_v4(const TeeDst<D>& ds, uint32_t off, const uint4& v) {
  dst_st_v4(ds.peers, off, v);
  dst_st_v4(ds.own, off, v);
}

// one item of an FP8 record -> its codes and the units of its buckets, with the loads of slice_fetch
template <int GPL>
__device__ __forceinline__ void full_unpack_fp8(const uint8_t* rec, const WarpItem& it, uint8_t* codes, float* scales) {
  uint32_t lo[GPL], hi[GPL];
  load_words<8, GPL>(rec + it.pay_off, 8, lo, hi);
  uint8_t* d = codes + lane_id() * (GPL * 8u);
  if ((reinterpret_cast<uintptr_t>(d) & 15u) == 0) {
#pragma unroll
    for (int k = 0; k < GPL; k += 2) st_v4(d + k * 8, make_uint4(lo[k], hi[k], lo[k + 1], hi[k + 1]));
  } else {
#pragma unroll
    for (int k = 0; k < GPL; ++k)
#pragma unroll
      for (int t = 0; t < 8; ++t) st_u8(d + k * 8 + t, ((t < 4 ? lo[k] : hi[k]) >> (8 * (t & 3))) & 0xFFu);
  }
  const uint32_t nb = item_n(it) >> (item_lpb_log2(it) + 3u);  // buckets of 8 << lg elements
  for (uint32_t b = lane_id(); b < nb; b += 32) scales[b] = __uint_as_float(ld_sys_u32(rec + it.meta_off + b * 8u));
}
// (inline: one definition across the translation units that include this header)
inline __device__ __noinline__ void bucket_unpack_fp8(const uint8_t* rec, const WarpItem it, uint8_t* codes, float* scales) {
  const uint32_t n = item_n(it);
  const uint32_t ng = div_up(n, 8u);
  if (lane_id() == 0) *scales = __uint_as_float(ld_sys_u32(rec + it.meta_off));
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    uint32_t lo, hi;
    load_word<8>(rec + it.pay_off, g, 8, lo, hi);
    uint8_t* d = codes + g * 8u;
    const uint32_t nv = min(8u, n - g * 8u);
    if (nv == 8u && (reinterpret_cast<uintptr_t>(d) & 7u) == 0) {
      st_v2(d, lo, hi);
    } else {
      for (uint32_t t = 0; t < nv; ++t) st_u8(d + t, ((t < 4 ? lo : hi) >> (8 * (t & 3))) & 0xFFu);
    }
  }
}
template <int GPL>
__device__ __forceinline__ void fp8_unpack_item(const uint8_t* rec, const WarpItem& it, uint8_t* codes, float* scales) {
  if (item_kind(it) == kItemFull)
    full_unpack_fp8<GPL>(rec, it, codes, scales);
  else
    bucket_unpack_fp8(rec, it, codes, scales);
}

// ======================================================================================
// FP8 in the sharded collectives (rs_kernel, ag_kernel and the generic reducers' item kernels).
// The sender prescales, then encodes as above; the all-gather's owner writes what every receiver
// decodes from the same codes; the reduce-scatter's owner adds each source's decoded value,
// fl(float(code) * unit), to its fp32 accumulator with a separate rounding (no FMA), in slot order.
// ======================================================================================
// full item, values in registers and already prescaled: publish meta + codes, and the decoded
// values to `out` (VEC: group aligned)
template <typename TO, int CODEC, int GPL, bool VEC, typename DST>
__device__ __forceinline__ void full_publish_fp8_x(const float (&x)[GPL][8], const WarpItem& it, const RngKey& rng,
                                                   const DST& ds, TO* __restrict__ out) {
  BucketMeta m[GPL];
  uint32_t lo[GPL], hi[GPL];
  full_send_fp8_codes<CODEC, GPL>(x, it, rng, ds, m, lo, hi);
  float d[GPL][8];
#pragma unroll
  for (int k = 0; k < GPL; ++k) fp8_decode8<CODEC>(lo[k], hi[k], m[k].unit, d[k]);
  slice_store<TO, GPL, VEC>(out, d);
}
// unaligned full item of src * prescale; SELF: also the decoded values to `self_out`
template <typename TS, typename TO, int CODEC, int GPL, bool SELF, typename DST>
__device__ __noinline__ void full_send_fp8_scaled_unaligned(const TS* __restrict__ src, const WarpItem it,
                                                            float prescale, const RngKey rng, const DST ds,
                                                            TO* __restrict__ self_out) {
  float x[GPL][8];
  slice_load_scalar<TS, GPL>(src, x);
  slice_scale<GPL>(x, prescale);
  if (SELF)
    full_publish_fp8_x<TO, CODEC, GPL, false>(x, it, rng, ds, self_out);
  else
    full_send_fp8_x<CODEC, GPL>(x, it, rng, ds);
}
// generic bucket item of src * prescale; self_out != nullptr: also the decoded values there
template <typename TS, typename TO, int CODEC, typename DST>
__device__ __noinline__ void bucket_send_fp8(const TS* __restrict__ src, const WarpItem it, float prescale,
                                             const RngKey rng, const DST ds, TO* __restrict__ self_out) {
  bucket_fp8_body<TS, TO, CODEC>(src, it, prescale, rng, ds, self_out);
}

// x = fl(x + fl(float(code) * unit)) for every source of the set, in slot order; the words of
// several sources are in flight at once, as in slice_accumulate
template <int CODEC, int GPL>
__device__ __forceinline__ void slice_accumulate_fp8(const SrcSet& ss, uint32_t meta_off, uint32_t pay_off,
                                                     uint32_t lg, float (&x)[GPL][8]) {
  const int cnt = ss.n - (ss.skip >= 0 ? 1 : 0);
  constexpr int kB = GPL == 4 ? 2 : 4;
  for (int i0 = 0; i0 < cnt; i0 += kB) {
    SliceWords<GPL> w[kB];
#pragma unroll
    for (int u = 0; u < kB; ++u) {
      // past the end: re-read the last source (its value is not added)
      const int i = min(i0 + u, cnt - 1);
      const int q = (ss.skip >= 0 && i >= ss.skip) ? i + 1 : i;
      slice_fetch<8, GPL>(ss.base + (size_t)q * ss.stride, meta_off, pay_off, lg, 8, w[u]);
    }
#pragma unroll
    for (int u = 0; u < kB; ++u) {
      if (i0 + u < cnt) {
#pragma unroll
        for (int k = 0; k < GPL; ++k) {
          float d[8];
          fp8_decode8<CODEC>(w[u].lo[k], w[u].hi[k], w[u].pm[k].unit, d);
#pragma unroll
          for (int j = 0; j < 8; ++j) x[k][j] = __fadd_rn(x[k][j], d[j]);
        }
      }
    }
  }
}

// reduce-scatter of a full item: my values * prescale + the decoded sources -> out (as full_rs_x)
template <typename T, int CODEC, int GPL, bool VEC>
__device__ __forceinline__ void full_rs_fp8_x(float (&x)[GPL][8], const WarpItem& it, float prescale,
                                              const SrcSet& ss, T* out) {
  slice_scale<GPL>(x, prescale);
  slice_accumulate_fp8<CODEC, GPL>(ss, it.meta_off, it.pay_off, item_lpb_log2(it), x);
  slice_store<T, GPL, VEC>(out, x);
}
template <typename T, int CODEC, int GPL>
__device__ __noinline__ void full_rs_fp8_unaligned(const T* src, const WarpItem it, float prescale, const SrcSet ss,
                                                   T* out) {
  float x[GPL][8];
  slice_load_scalar<T, GPL>(src, x);
  full_rs_fp8_x<T, CODEC, GPL, false>(x, it, prescale, ss, out);
}

// x[8] of group g += the decoded values of every source of the set (slot order)
template <int CODEC>
__device__ __forceinline__ void bucket_add_sources_fp8(const SrcSet& ss, const WarpItem& it, uint32_t g,
                                                       float (&x)[8]) {
  for (int q = 0; q < ss.n; ++q) {
    if (q == ss.skip) continue;
    const uint8_t* rec = ss.base + (size_t)q * ss.stride;
    uint32_t lo, hi;
    load_word<0>(rec + it.pay_off, g, 8, lo, hi);
    float d[8];
    fp8_decode8<CODEC>(lo, hi, __uint_as_float(ld_sys_v2(rec + it.meta_off).x), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = __fadd_rn(x[j], d[j]);
  }
}
template <typename T, int CODEC>
__device__ __noinline__ void bucket_rs_fp8(const T* src, const WarpItem it, float prescale, const SrcSet ss, T* out) {
  const uint32_t n = item_n(it);
  const uint32_t ng = div_up(n, 8u);
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
    int nv;
    bucket_load_group<T>(src, g, n, prescale, x, nv);
    bucket_add_sources_fp8<CODEC>(ss, it, g, x);
    store8_scalar<T>(out + g * 8u, nv, x);
  }
}

// ======================================================================================
// FP8 in the allreduce (sra_kernel phase B, oneshot_kernel phase 2). Phase B sums as the
// reduce-scatter does -- my values * prescale, then fl(float(code) * unit) of every source in slot
// order, each add rounded on its own -- encodes the fp32 sum once, publishes meta + codes and writes
// the values decoded from its own codes to `blk`, so every rank ends with the same bytes. The
// one-shot receiver sums the decoded values of every source, its own included, from +0.
// ======================================================================================
template <typename T, int CODEC, int GPL, bool VEC, typename DST>
__device__ __forceinline__ void full_reduce_fp8_x(float (&x)[GPL][8], T* __restrict__ blk, const WarpItem& it,
                                                  float prescale, const RngKey& rng, const SrcSet& ss, const DST& ds) {
  slice_scale<GPL>(x, prescale);
  slice_accumulate_fp8<CODEC, GPL>(ss, it.meta_off, it.pay_off, item_lpb_log2(it), x);
  full_publish_fp8_x<T, CODEC, GPL, VEC>(x, it, rng, ds, blk);
}
template <typename T, int CODEC, int GPL, typename DST>
__device__ __noinline__ void full_reduce_fp8_unaligned(T* __restrict__ blk, const WarpItem it, float prescale,
                                                       const RngKey rng, const SrcSet ss, const DST ds) {
  float x[GPL][8];
  slice_load_scalar<T, GPL>(blk, x);
  full_reduce_fp8_x<T, CODEC, GPL, false>(x, blk, it, prescale, rng, ss, ds);
}

// generic bucket item: two passes (min/max of the sums, then encode), as bucket_quantize; every
// lane reads a group of `blk` before it writes the same group
template <typename T, int CODEC, typename DST>
__device__ __noinline__ void bucket_reduce_fp8(T* __restrict__ blk, const WarpItem it, float prescale,
                                               const RngKey rng, const SrcSet ss, const DST ds) {
  const uint32_t n = item_n(it);
  const uint32_t ng = div_up(n, 8u);
  float mn = CGX_INF_POS, mx = CGX_INF_NEG;
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
    int nv;
    bucket_load_group<T>(blk, g, n, prescale, x, nv);
    bucket_add_sources_fp8<CODEC>(ss, it, g, x);
    minmax8_pred(x, nv, mn, mx);
  }
  warp_minmax(mn, mx);
  const BucketMeta m = fp8_meta(mn, mx, CODEC);
  const float inv = fp8_inv_unit(m.unit, CODEC);
  const DST du = unicast_of(ds);
  if (lane_id() == 0) dst_st_v2(du, it.meta_off, __float_as_uint(m.unit), __float_as_uint(m.min));
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
    int nv;
    bucket_load_group<T>(blk, g, n, prescale, x, nv);
    bucket_add_sources_fp8<CODEC>(ss, it, g, x);
    uint32_t lo, hi;
    fp8_encode8<CODEC>(x, inv, rng, it.elem_off + g * 8u, lo, hi);
    const uint64_t w = ((uint64_t)hi << 32 | lo) & (nv >= 8 ? ~0ull : (1ull << (8 * nv)) - 1ull);
    const uint32_t o = it.pay_off + g * 8u;
    for (int t = 0; t < 8; ++t) dst_st_u8(du, o + t, (uint32_t)(w >> (8 * t)) & 0xFFu);
    float dec[8];
    fp8_decode8<CODEC>(lo, hi, m.unit, dec);
    store8_scalar<T>(blk + g * 8u, nv, dec);
  }
}

// out = sum of the decoded values of all sources, slot order, from +0 (one-shot phase 2)
template <typename TO, int CODEC, int GPL, bool VEC>
__device__ __forceinline__ void full_recv_sum_fp8(const SrcSet& ss, const WarpItem& it, TO* __restrict__ out) {
  float x[GPL][8];
#pragma unroll
  for (int k = 0; k < GPL; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) x[k][j] = 0.f;
  slice_accumulate_fp8<CODEC, GPL>(ss, it.meta_off, it.pay_off, item_lpb_log2(it), x);
  slice_store<TO, GPL, VEC>(out, x);
}
template <typename TO, int CODEC, int GPL>
__device__ __noinline__ void full_recv_sum_fp8_unaligned(const SrcSet ss, const WarpItem it, TO* __restrict__ out) {
  full_recv_sum_fp8<TO, CODEC, GPL, false>(ss, it, out);
}
template <typename TO, int CODEC>
__device__ __noinline__ void bucket_recv_sum_fp8(const SrcSet ss, const WarpItem it, TO* __restrict__ out) {
  const uint32_t n = item_n(it);
  const uint32_t ng = div_up(n, 8u);
  for (uint32_t g = lane_id(); g < ng; g += 32) {
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = 0.f;
    bucket_add_sources_fp8<CODEC>(ss, it, g, x);
    store8_scalar<TO>(out + g * 8u, (int)min(8u, n - g * 8u), x);
  }
}

}  // namespace dev
}  // namespace cgx

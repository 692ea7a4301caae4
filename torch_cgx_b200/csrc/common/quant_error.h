// Quantization-error estimate of a layer table at several bit widths (adaptive per-layer widths).
//
// For every layer and every candidate width b the estimate is the squared error that one
// quantization round trip at b bits would add to the layer:
//   deterministic  sum_i (decode(encode(x_i)) - x_i)^2, with the per-bucket min/max, make_meta,
//                  inv_unit, encode_level and decode_level of quant_math.h, i.e. exactly the levels
//                  the quantizer sends;
//   stochastic     the expected squared error of QSGD rounding, sum_i unit^2 * f_i * (1 - f_i) with
//                  f_i = frac((x_i - min) * inv); computed as unit^2 * sum_i f_i * (1 - f_i).
// x_i is the fp32 value the encoder sees (dtype conversion, then * prescale). A bucket whose
// max - min is not finite (NaN or Inf inside, or an overflowing range) decodes to non-finite values
// on the wire; its error is NaN at every width. With skip_incomplete the incomplete tail bucket of a
// layer travels raw and contributes 0.
//
// Summation order (the same on the CPU and in kernels/quant_error.cu, so both give the same bits):
// inside a bucket, "lane" l = g % 32 of pack group g (8 elements) sums its groups in order in fp32,
// then the 32 lane sums are combined by an xor butterfly (strides 16, 8, 4, 2, 1). The fp32 bucket
// partials go into the fp64 layer total the same way: bucket j of the layer to lane j % 32, in order,
// then the butterfly.
//
// Sharded mode (a reduce-scatter input): the tensor holds `chunks` copies of one shard's layer table
// at stride S = numel / chunks, and chunk `skip_chunk` (the receiving rank's own, -1 for none) is
// left out. Row l is the error of layer l summed over the included chunks: its fp32 bucket partials
// form one list, chunk-major (included chunks in increasing order), then bucket, and list entry i
// goes to lane i % 32 in order, then the butterfly. With chunks = 1 the list is the layer's buckets.
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>
#include "block_ops.h"
#include "quant_math.h"
#include "wire.h"

namespace cgx {

constexpr int kQErrMaxCandidates = 8;
constexpr int kQErrLanes = 32;

struct alignas(8) QErrLayer {
  uint64_t elem_off;
  uint64_t numel;   // elements that are quantized: the whole layer, or its complete buckets (skip_incomplete)
  uint32_t bucket;  // already clamped to [1, kMaxBlockElems]
  uint32_t unused;
};

// Buckets of every layer, flattened in layer order: layer l owns buckets [first[l], first[l + 1]).
// Bucket j of layer l covers elements [elem_off + j * bucket, min(elem_off + numel, ... + bucket)).
inline std::vector<uint64_t> qerr_first(const std::vector<QErrLayer>& layers) {
  std::vector<uint64_t> first(layers.size() + 1, 0);
  for (size_t l = 0; l < layers.size(); ++l)
    first[l + 1] = first[l] + (layers[l].numel + layers[l].bucket - 1) / layers[l].bucket;
  return first;
}

// Per-candidate quantities of a bucket with finite range.
struct QErrCand {
  float unit, inv, maxlvl;
};

namespace cpu {

// xor butterfly over 32 lane values (strides 16 .. 1), as __shfl_xor_sync computes it; returns lane 0's
template <typename F>
inline F lane_butterfly(F (&v)[kQErrLanes]) {
  for (int s = kQErrLanes / 2; s >= 1; s /= 2) {
    F next[kQErrLanes];
    for (int l = 0; l < kQErrLanes; ++l) next[l] = v[l] + v[l ^ s];
    for (int l = 0; l < kQErrLanes; ++l) v[l] = next[l];
  }
  return v[0];
}

// fp32 partials of one bucket (n prescaled values) for each of the K candidates.
inline void bucket_quantization_error(const float* x, uint32_t n, const int* bits, int K, bool stochastic,
                                      float* out) {
  float mn = x[0], mx = x[0];
  for (uint32_t i = 1; i < n; ++i) {
    mn = nan_min(mn, x[i]);
    mx = nan_max(mx, x[i]);
  }
  if (!std::isfinite(mx - mn)) {
    for (int k = 0; k < K; ++k) out[k] = canonical_nan();
    return;
  }
  QErrCand c[kQErrMaxCandidates];
  for (int k = 0; k < K; ++k) {
    const BucketMeta m = make_meta(mn, mx, bits[k]);
    c[k] = {m.unit, inv_unit(m.unit), (float)max_level(bits[k])};
  }
  float lane[kQErrMaxCandidates][kQErrLanes] = {};
  const uint32_t groups = div_up(n, 8u);
  for (uint32_t g = 0; g < groups; ++g) {
    for (uint32_t i = g * 8u; i < g * 8u + 8u && i < n; ++i) {
      const float d = x[i] - mn;
      for (int k = 0; k < K; ++k) {
        float e;
        if (stochastic) {
          const float t = d * c[k].inv;
          const float f = t - std::floor(t);
          e = f * (1.0f - f);
        } else {
          const float r = decode_level(encode_level(x[i], mn, c[k].inv, 0.5f, c[k].maxlvl), c[k].unit, mn) - x[i];
          e = r * r;
        }
        lane[k][g % kQErrLanes] += e;
      }
    }
  }
  for (int k = 0; k < K; ++k) {
    const float sum = lane_butterfly(lane[k]);
    out[k] = stochastic ? (c[k].unit * c[k].unit) * sum : sum;
  }
}

// out[l * K + k]: the error of layer l at bits[k] (see the top of this file), summed over chunks
// 0..chunks-1 at stride chunk_stride except skip_chunk (-1: none).
inline void quantization_error(const void* t, int dtype, const std::vector<QErrLayer>& layers, const int* bits,
                               int K, bool stochastic, float prescale, double* out, int chunks = 1,
                               uint64_t chunk_stride = 0, int skip_chunk = -1) {
  std::vector<float> x(kMaxBlockElems);
  float part[kQErrMaxCandidates];
  for (size_t l = 0; l < layers.size(); ++l) {
    const QErrLayer& L = layers[l];
    double tot[kQErrMaxCandidates][kQErrLanes] = {};
    uint64_t j = 0;  // position in the layer's chunk-major list of bucket partials
    for (int c = 0; c < chunks; ++c) {
      if (c == skip_chunk) continue;
      const uint64_t base = (uint64_t)c * chunk_stride + L.elem_off;
      for (uint64_t o = 0; o < L.numel; o += L.bucket, ++j) {
        const uint32_t n = (uint32_t)(L.numel - o < L.bucket ? L.numel - o : L.bucket);
        for (uint32_t i = 0; i < n; ++i) x[i] = load_elem(t, dtype, base + o + i) * prescale;
        bucket_quantization_error(x.data(), n, bits, K, stochastic, part);
        for (int k = 0; k < K; ++k) tot[k][j % kQErrLanes] += (double)part[k];
      }
    }
    for (int k = 0; k < K; ++k) out[l * K + k] = lane_butterfly(tot[k]);
  }
}

}  // namespace cpu
}  // namespace cgx

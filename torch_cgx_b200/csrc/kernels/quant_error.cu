// Quantization-error estimate (common/quant_error.h) of a layer table at up to 8 bit widths in
// one pass over the gradient.
//
// qerr_buckets: one warp per quantization bucket of the flattened bucket list (the host uploads only
// the layer table and each layer's first bucket; a warp finds its layer by binary search). Pass 1 loads the
// bucket for its min/max (minmax8 trees, warp_minmax: the meta the fused kernel would send);
// pass 2 loads it again -- from L1/L2, the bucket is at most 32 KB -- and accumulates the error of
// every candidate in one fp32 register each. Levels come from level_magic, bit for bit
// encode_level(); the fp32 lane sums are combined by an xor butterfly. 16-byte loads when the
// bucket is group aligned, scalar loads otherwise.
// qerr_layers: one warp per (layer, candidate) adds the bucket partials into the fp64 layer total:
// lane j % 32 takes bucket j in order, then an xor butterfly. No atomics: the result is the same bits
// on every run, and the CPU's.
//
// Sharded mode (a reduce-scatter input: `chunks` copies of one shard's table at stride S, chunk
// skip_chunk left out): qerr_buckets' index space is (included chunk j, shard bucket), b = j * nb +
// bucket; the chunk is j, or j + 1 from skip_chunk on. qerr_layers reads layer l's partials as one
// list, chunk-major then bucket, and lane i % 32 takes list entry i in order. With chunks = 1 both
// are the single-chunk kernels above, bit for bit.
#include "../common/quant_error.h"
#include "item_path.cuh"
#include "launch.h"

namespace cgx {
using namespace dev;

namespace {
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int K8 = kQErrMaxCandidates;

template <typename T, bool VEC>
__device__ __forceinline__ void load_group(const T* p, uint32_t nv, float prescale, float (&x)[8]) {
  if (VEC && nv == 8)
    load8_vec<T>(p, x);
  else
    load8_scalar<T>(p, (int)nv, x);
  if (prescale != 1.0f) {
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = __fmul_rn(x[j], prescale);
  }
}

template <typename T, bool VEC, bool STOCH>
__device__ __forceinline__ void bucket_error(const T* __restrict__ p, uint32_t n, float prescale, const int* bits,
                                             int K, float* __restrict__ out) {
  const uint32_t groups = div_up(n, 8u);
  const uint32_t lane = lane_id();
  float mn = CGX_INF_POS, mx = CGX_INF_NEG;
#pragma unroll 2
  for (uint32_t g = lane; g < groups; g += 32u) {
    const uint32_t nv = min(8u, n - g * 8u);
    float x[8];
    load_group<T, VEC>(p + g * 8u, nv, prescale, x);
    if (nv == 8)
      minmax8(x, mn, mx);
    else
      minmax8_pred(x, (int)nv, mn, mx);
  }
  warp_minmax(mn, mx);
  if (!isfinite(__fsub_rn(mx, mn))) {
    if (lane < (uint32_t)K) out[lane] = __int_as_float((int)kCanonicalNaNBits);
    return;
  }
  QErrCand c[K8];
  float acc[K8];
#pragma unroll
  for (int k = 0; k < K8; ++k) {
    const int b = k < K ? bits[k] : 8;
    const BucketMeta m = make_meta(mn, mx, b);
    c[k] = {m.unit, inv_unit(m.unit), (float)max_level(b)};
    acc[k] = 0.f;
  }
#pragma unroll 1
  for (uint32_t g = lane; g < groups; g += 32u) {
    const uint32_t nv = min(8u, n - g * 8u);
    float x[8];
    load_group<T, VEC>(p + g * 8u, nv, prescale, x);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if ((uint32_t)j < nv) {
        const float d = __fsub_rn(x[j], mn);
#pragma unroll
        for (int k = 0; k < K8; ++k) {
          if (k < K) {
            float e;
            if (STOCH) {
              const float t = __fmul_rn(d, c[k].inv);
              const float f = __fsub_rn(t, floorf(t));
              e = __fmul_rn(f, __fsub_rn(1.0f, f));
            } else {
              // every bucket here has a finite range: the clamp of encode_level is a no-op
              const float q = __fsub_rn(level_magic<false>(x[j], mn, c[k].inv, 0.5f, c[k].maxlvl), CGX_MAGIC);
              const float r = __fsub_rn(__fmaf_rn(c[k].unit, q, mn), x[j]);
              e = __fmul_rn(r, r);
            }
            acc[k] = __fadd_rn(acc[k], e);
          }
        }
      }
    }
  }
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1)
#pragma unroll
    for (int k = 0; k < K8; ++k)
      if (k < K) acc[k] = __fadd_rn(acc[k], __shfl_xor_sync(kAll, acc[k], s));
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K8; ++k)
      if (k < K) out[k] = STOCH ? __fmul_rn(__fmul_rn(c[k].unit, c[k].unit), acc[k]) : acc[k];
  }
}

struct Cands {
  int bits[K8];
};

template <typename T, bool STOCH>
__global__ void __launch_bounds__(kThreads) qerr_buckets(const T* __restrict__ t, const QErrLayer* __restrict__ layers,
                                                         const uint64_t* __restrict__ first, int L, uint64_t nb,
                                                         uint64_t total, uint64_t stride, int skip, Cands cands, int K,
                                                         float prescale, float* __restrict__ partial) {
  const uint64_t b = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (b >= total) return;
  const uint64_t j = b / nb, sb = b - j * nb;  // included chunk, bucket of the shard table
  const uint64_t c = (skip >= 0 && j >= (uint64_t)skip) ? j + 1 : j;
  int lo = 0, hi = L - 1;  // the layer l with first[l] <= sb < first[l + 1]
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= sb)
      lo = mid;
    else
      hi = mid - 1;
  }
  const QErrLayer ly = layers[lo];
  const uint64_t o = (sb - first[lo]) * ly.bucket;
  const uint64_t left = ly.numel - o;
  const uint32_t n = left < ly.bucket ? (uint32_t)left : ly.bucket;
  const T* p = t + c * stride + ly.elem_off + o;
  float* out = partial + b * (uint64_t)K;
  if (group_aligned<T>(p))
    bucket_error<T, true, STOCH>(p, n, prescale, cands.bits, K, out);
  else
    bucket_error<T, false, STOCH>(p, n, prescale, cands.bits, K, out);
}

__global__ void __launch_bounds__(kThreads) qerr_layers(const float* __restrict__ partial,
                                                        const uint64_t* __restrict__ first, int L, int K,
                                                        uint64_t nb, uint64_t included, double* __restrict__ out) {
  const int i = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (i >= L * K) return;
  const int l = i / K, k = i % K;
  const uint64_t f = first[l], nbl = first[l + 1] - f, len = included * nbl;
  double acc = 0.0;
  for (uint64_t e = lane_id(); e < len; e += 32u) {  // entry e of the chunk-major list: chunk e / nbl
    const uint64_t j = e / nbl;
    acc += (double)partial[(j * nb + f + (e - j * nbl)) * (uint64_t)K + (uint64_t)k];
  }
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) acc += __shfl_xor_sync(kAll, acc, s);
  if (lane_id() == 0) out[i] = acc;
}

uint64_t included_chunks(const QErrArgs& a) {
  return (uint64_t)a.chunks - (a.skip_chunk >= 0 ? 1u : 0u);
}

template <typename T>
void launch_buckets(const QErrArgs& a, const Cands& c, cudaStream_t s) {
  const uint64_t total = included_chunks(a) * a.nbuckets;
  const unsigned blocks = (unsigned)((total + kWarps - 1) / kWarps);
  const T* t = static_cast<const T*>(a.data);
  if (a.stochastic)
    qerr_buckets<T, true><<<blocks, kThreads, 0, s>>>(t, a.layer_table, a.first, a.layers, a.nbuckets, total,
                                                      a.chunk_stride, a.skip_chunk, c, a.K, a.prescale, a.partial);
  else
    qerr_buckets<T, false><<<blocks, kThreads, 0, s>>>(t, a.layer_table, a.first, a.layers, a.nbuckets, total,
                                                       a.chunk_stride, a.skip_chunk, c, a.K, a.prescale, a.partial);
}
}  // namespace

cudaError_t launch_quantization_error(const QErrArgs& a, cudaStream_t stream) {
  if (a.K < 1 || a.K > K8) return cudaErrorInvalidValue;
  if (a.chunks < 1 || a.skip_chunk < -1 || a.skip_chunk >= a.chunks) return cudaErrorInvalidValue;
  if (a.nbuckets > 0 && included_chunks(a) > 0) {
    Cands c;
    for (int k = 0; k < K8; ++k) c.bits[k] = k < a.K ? a.bits[k] : 8;
    switch (a.dtype) {
      case kF32: launch_buckets<float>(a, c, stream); break;
      case kF16: launch_buckets<__half>(a, c, stream); break;
      default: launch_buckets<__nv_bfloat16>(a, c, stream); break;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  if (a.layers > 0) {
    const int n = a.layers * a.K;
    qerr_layers<<<(n + kWarps - 1) / kWarps, kThreads, 0, stream>>>(a.partial, a.first, a.layers, a.K, a.nbuckets,
                                                                     included_chunks(a), a.out);
  }
  return cudaGetLastError();
}

}  // namespace cgx

// The cross-node stage of the compressed all-to-all (DESIGN §2.13f): one launch quantizes every
// chunk a rank sends to the ranks of other nodes into one contiguous send buffer, and one launch
// decodes every chunk it received from them into its rows of the output.
//
// A chunk's record is exactly what Reducer::all_to_all sends for it: the one-layer geometry of
// common/a2a.h, buckets counted from the chunk's first element, encoded and decoded by the same
// warp-item primitives as a2a_kernel. Nothing is planned or uploaded: the launch gets each chunk's
// element count, offsets and peer in its parameters, and warp t of the whole grid derives item t
// from them. The items of all chunks are numbered consecutively (item_first), so a launch balances
// over every chunk whatever the splits.
#include "a2a_kernel.cuh"

namespace cgx {
namespace dev {

// item t of the launch: its chunk, the item, and the byte offset of its block's record in the buffer
template <typename T>
__device__ __forceinline__ int a2a_remote_item(const A2aRemoteParams& p, uint32_t t, WarpItem& it, uint64_t& rec) {
  int lo = 0, hi = p.nchunks - 1;  // the chunk i with item_first[i] <= t < item_first[i + 1]
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.item_first[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const A2aGeom g = a2a_geom(p.cnt[lo], p.bits, p.bucket, (int)sizeof(T));
  const uint32_t u = t - p.item_first[lo], b = u / g.block_items;
  it = a2a_block_item(g, b, u - b * g.block_items);
  rec = p.wire_off[lo] + (uint64_t)b * g.block_wire;
  return lo;
}

template <typename T, int KB, int GPL, int CODEC>
__global__ void __launch_bounds__(kSraThreads) a2a_pack_kernel(const __grid_constant__ A2aRemoteParams p) {
  const SrcSet no_src{nullptr, 0u, 0, -1};
  const uint32_t warps = gridDim.x * kSraWarps;
  for (uint32_t t = blockIdx.x * kSraWarps + (threadIdx.x >> 5); t < p.item_first[p.nchunks]; t += warps) {
    WarpItem it;
    uint64_t rec;
    const int i = a2a_remote_item<T>(p, t, it, rec);
    const T* src = reinterpret_cast<const T*>(p.in) + p.elem_off[i] + it.elem_off;
    const OneDst push{reinterpret_cast<uint8_t*>(p.out) + rec};
    RngKey rng = p.rng;
    rng.stream = a2a_rng_stream(p.rank, p.peer[i]);
    if constexpr (CODEC != kMaxMin) {
      a2a_send_item_fp8<T, CODEC, GPL, OneDst>(src, it, rng, push);
      continue;
    }
    if (item_kind(it) == kItemFull) {
      if (group_aligned<T>(src)) {
        float x[GPL][8];
        slice_load_vec<T, GPL>(src, x);
        full_send_x<T, KB, GPL, false, true>(x, it, 1.0f, rng, push, (T*)nullptr);
      } else {
        full_send_unaligned<T, T, KB, GPL, false>(src, it, 1.0f, rng, push, (T*)nullptr);
      }
    } else {
      bucket_quantize<T, T>(src, it, 1.0f, rng, no_src, push, (T*)nullptr);
    }
  }
}

// CODES: the records are unpacked into one FP8 code byte per element (p.out) and the units of their
// buckets (p.out_scales[e / bucket] for the bucket starting at output element e)
template <typename T, int KB, int GPL, int CODEC, bool CODES>
__global__ void __launch_bounds__(kSraThreads) a2a_unpack_kernel(const __grid_constant__ A2aRemoteParams p) {
  const uint32_t warps = gridDim.x * kSraWarps;
  for (uint32_t t = blockIdx.x * kSraWarps + (threadIdx.x >> 5); t < p.item_first[p.nchunks]; t += warps) {
    WarpItem it;
    uint64_t rec;
    const int i = a2a_remote_item<T>(p, t, it, rec);
    const uint8_t* base = reinterpret_cast<const uint8_t*>(p.in) + rec;
    const uint64_t e = p.elem_off[i] + it.elem_off;
    if constexpr (CODES) {
      fp8_unpack_item<GPL>(base, it, reinterpret_cast<uint8_t*>(p.out) + e, p.out_scales + e / p.bucket);
      continue;
    }
    T* dst = reinterpret_cast<T*>(p.out) + e;
    if constexpr (CODEC != kMaxMin) {
      a2a_recv_item_fp8<T, CODEC, GPL>(base, it, dst);
      continue;
    }
    const SrcSet ss{base, 0u, 1, -1};
    if (item_kind(it) == kItemFull) {
      if (group_aligned<T>(dst)) {
        SliceWords<GPL> sw;
        slice_fetch<KB, GPL>(ss.base, it.meta_off, it.pay_off, item_lpb_log2(it), KB ? KB : item_bits(it), sw);
        full_recv_w<T, KB, GPL, true>(sw, it, dst);
      } else {
        full_recv_unaligned<T, KB, GPL>(ss, it, dst);
      }
    } else {
      bucket_recv<T>(ss, it, dst);
    }
  }
}

}  // namespace dev

namespace {

int a2a_remote_grid(uint32_t items) {
  // initialized once, thread-safe: the ranks of one process may launch from several threads
  static const int sms = [] {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      return 132;
    return n;
  }();
  // one warp per item; enough CTAs to fill every SM a few times over, the rest is grid-stride
  const uint32_t want = (items + kSraWarps - 1) / kSraWarps;
  return (int)(want < (uint32_t)sms * 8u ? want : (uint32_t)sms * 8u);
}

template <typename T, int GPL>
cudaError_t launch_pack_gpl(const A2aRemoteParams& p, int grid, cudaStream_t s) {
  if (p.codec != kMaxMin) {
    return dispatch_fp8(p.codec, cudaErrorInvalidValue, [&](auto c) {
      dev::a2a_pack_kernel<T, 8, GPL, decltype(c)::value><<<grid, kSraThreads, 0, s>>>(p);
      return cudaGetLastError();
    });
  } else {
    switch (p.bits) {
      case 2: dev::a2a_pack_kernel<T, 2, GPL, kMaxMin><<<grid, kSraThreads, 0, s>>>(p); break;
      case 4: dev::a2a_pack_kernel<T, 4, GPL, kMaxMin><<<grid, kSraThreads, 0, s>>>(p); break;
      case 8: dev::a2a_pack_kernel<T, 8, GPL, kMaxMin><<<grid, kSraThreads, 0, s>>>(p); break;
      default: dev::a2a_pack_kernel<T, 0, GPL, kMaxMin><<<grid, kSraThreads, 0, s>>>(p); break;
    }
  }
  return cudaGetLastError();
}

template <typename T, int GPL>
cudaError_t launch_unpack_gpl(const A2aRemoteParams& p, int grid, cudaStream_t s) {
  const bool codes = p.out_scales != nullptr;
  if (p.codec != kMaxMin) {
    return dispatch_fp8(p.codec, cudaErrorInvalidValue, [&](auto c) {
      if (codes)
        dev::a2a_unpack_kernel<T, 8, GPL, decltype(c)::value, true><<<grid, kSraThreads, 0, s>>>(p);
      else
        dev::a2a_unpack_kernel<T, 8, GPL, decltype(c)::value, false><<<grid, kSraThreads, 0, s>>>(p);
      return cudaGetLastError();
    });
  } else {
    switch (p.bits) {
      case 2: dev::a2a_unpack_kernel<T, 2, GPL, kMaxMin, false><<<grid, kSraThreads, 0, s>>>(p); break;
      case 4: dev::a2a_unpack_kernel<T, 4, GPL, kMaxMin, false><<<grid, kSraThreads, 0, s>>>(p); break;
      case 8: dev::a2a_unpack_kernel<T, 8, GPL, kMaxMin, false><<<grid, kSraThreads, 0, s>>>(p); break;
      default: dev::a2a_unpack_kernel<T, 0, GPL, kMaxMin, false><<<grid, kSraThreads, 0, s>>>(p); break;
    }
  }
  return cudaGetLastError();
}

template <int GPL>
cudaError_t launch_remote_gpl(const A2aRemoteParams& p, bool pack, int grid, cudaStream_t s) {
  switch (p.dtype) {
    case kF32: return pack ? launch_pack_gpl<float, GPL>(p, grid, s) : launch_unpack_gpl<float, GPL>(p, grid, s);
    case kF16: return pack ? launch_pack_gpl<__half, GPL>(p, grid, s) : launch_unpack_gpl<__half, GPL>(p, grid, s);
    case kBF16:
      return pack ? launch_pack_gpl<__nv_bfloat16, GPL>(p, grid, s) : launch_unpack_gpl<__nv_bfloat16, GPL>(p, grid, s);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_remote(const A2aRemoteParams& p, bool pack, cudaStream_t s) {
  if (p.nchunks < 0 || p.nchunks > kA2aMaxWorld || p.bits < 1 || p.bits > 8 ||
      (p.codec != kMaxMin && p.bits != 8) || (!pack && p.out_scales != nullptr && p.codec == kMaxMin))
    return cudaErrorInvalidValue;
  if (p.nchunks == 0 || p.item_first[p.nchunks] == 0) return cudaSuccess;
  const int grid = a2a_remote_grid(p.item_first[p.nchunks]);
  return a2a_slice_elems(p.bits, p.bucket) == 1024u ? launch_remote_gpl<4>(p, pack, grid, s)
                                                    : launch_remote_gpl<2>(p, pack, grid, s);
}

}  // namespace

cudaError_t launch_a2a_pack(const A2aRemoteParams& p, cudaStream_t stream) { return launch_remote(p, true, stream); }
cudaError_t launch_a2a_unpack(const A2aRemoteParams& p, cudaStream_t stream) { return launch_remote(p, false, stream); }

}  // namespace cgx

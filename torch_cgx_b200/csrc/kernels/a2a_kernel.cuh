// Compressed all-to-all: every rank quantizes its chunk for rank q once, pushes it into q's recv1
// slot for this rank and decodes the chunks that arrive into its output rows. No reduction, no
// requantization. Instantiated in translation units of its own (a2a_{f32,f16,bf16}.cu) for the
// reason given at launch_sra_inst.
//
// Splits differ per pair and change every call, and a rank knows only its own row and column of
// the split matrix. So nothing is planned on the host: a pair's blocks, items and windows are a
// function of (elements, bits, bucket, dtype) (common/a2a.h) that both ends evaluate.
//
// Lane c of a pair carries the chunk's blocks c, c + G, ... through its share of the slot, in
// windows of `bpw` blocks. The kernel runs in rounds k = 0, 1, ...; in round k lane c
//   1. waits until every destination that still has a window k released window k - 1,
//   2. quantizes and pushes window k to each of them, then releases a "landed" flag to each,
//   3. waits for window k of every source that still has one, decodes it, and releases a
//      "released" flag to each.
// Both ends of a pair know its window count, so each rank stops after its own last window. Round k
// of a rank waits only for round k - 1 (step 1) or round k (step 3, whose step 2 needs round k - 1)
// of its peers, so by induction every round completes. Flag values are (epoch << 32) | (k + 1),
// 64-bit, from the device-side epoch: no host state, and graph replays stay correct.
// The kernel ends with rs_kernel's handshake on flags2, so the next call of any kind may reuse the
// slots (docs/MEMORY_MODEL.md).
#pragma once
#include "../common/a2a.h"
#include "combine.cuh"
#include "sra_kernels.cuh"

namespace cgx {
namespace dev {

__device__ __forceinline__ uint64_t a2a_tag(uint32_t epoch, uint32_t k) {
  return ((uint64_t)epoch << 32) | (uint64_t)(k + 1u);
}
__device__ __forceinline__ void st_release_sys_u64(uint64_t* flag, uint64_t v) {
  asm volatile("fence.acq_rel.sys;\n\tst.relaxed.sys.global.u64 [%0], %1;" ::"l"(flag), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys_u64(const uint64_t* flag) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flag) : "memory");
  return v;
}
// wait_flag for the 64-bit window flags: 0 reached, 1 timeout, 2 abort
__device__ __forceinline__ int wait_flag_u64(const uint64_t* flag, uint64_t target, uint64_t timeout_ns,
                                             const uint32_t* abort_word) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while ((int64_t)(ld_acquire_sys_u64(flag) - target) < 0) {
    if ((++spins & 0x3FFu) == 0) {
      if (abort_word != nullptr && *reinterpret_cast<const volatile uint32_t*>(abort_word) != 0) return 2;
      const uint64_t now = globaltimer_ns();
      if (t0 == 0)
        t0 = now;
      else if (now - t0 > timeout_ns)
        return 1;
    }
  }
  return 0;
}

// warp 0, warp lane q: wait for my flag of peer q when `need`; false on timeout / abort (recorded in
// the status word with the peer and the lane, as wait_peers does)
__device__ __forceinline__ bool a2a_wait(const A2aParams& p, const uint64_t* my_flags, bool need, uint64_t target,
                                         uint32_t code) {
  const uint32_t q = lane_id();
  int rc = 0;
  if (need) {
    rc = wait_flag_u64(my_flags + (size_t)q * p.flag_stride + blockIdx.x, target, p.timeout_ns, p.abort_word);
    if (rc != 0) *p.status = (rc == 2 ? (uint32_t)kSraAborted : code) | (q << 8) | ((uint32_t)blockIdx.x << 16);
  }
  return __all_sync(kAll, rc == 0);
}

// The scaled send (SCALE): the values T(x * s) of one row, 16 bytes or one element at a time
template <typename T>
__device__ __forceinline__ uint4 scale_round16(const uint4& raw, float s) {
  float x[DT<T>::kVec];
  unpack16<T>(raw, x);
#pragma unroll
  for (int i = 0; i < DT<T>::kVec; ++i) x[i] = scale_round<T>(x[i], s);
  return pack16<T>(x);
}
__device__ __forceinline__ uint32_t elem_bits(float v) { return __float_as_uint(v); }
__device__ __forceinline__ uint32_t elem_bits(__half v) { return __half_as_ushort(v); }
__device__ __forceinline__ uint32_t elem_bits(__nv_bfloat16 v) { return __bfloat16_as_ushort(v); }
template <int GPL, typename T>
__device__ __forceinline__ void slice_scale_round(float (&x)[GPL][8], float s) {
#pragma unroll
  for (int k = 0; k < GPL; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) x[k][j] = scale_round<T>(x[k][j], s);
}

// raw items travel as the T bits, unchanged (a NaN keeps its payload, -0 stays -0)
template <typename T>
__device__ __forceinline__ void a2a_raw_send(const T* src, const WarpItem& it, uint8_t* slot) {
  const uint32_t n = item_n(it);
  uint8_t* dst = slot + it.meta_off;
  uint32_t done = 0;
  if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
    const uint32_t vecs = n * (uint32_t)sizeof(T) / 16u;
    for (uint32_t v = lane_id(); v < vecs; v += 32) st_v4(dst + v * 16u, reinterpret_cast<const uint4*>(src)[v]);
    done = vecs * 16u / (uint32_t)sizeof(T);
  }
  for (uint32_t i = done + lane_id(); i < n; i += 32) {
    if (sizeof(T) == 4)
      st_u32(dst + i * 4u, reinterpret_cast<const uint32_t*>(src)[i]);
    else
      st_u16(dst + i * 2u, reinterpret_cast<const uint16_t*>(src)[i]);
  }
}
// the same for the bits of T(x * s) (SCALE)
template <typename T>
__device__ __forceinline__ void a2a_raw_send_scaled(const T* src, const WarpItem& it, uint8_t* slot, float s) {
  const uint32_t n = item_n(it);
  uint8_t* dst = slot + it.meta_off;
  uint32_t done = 0;
  if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
    const uint32_t vecs = n * (uint32_t)sizeof(T) / 16u;
    for (uint32_t v = lane_id(); v < vecs; v += 32)
      st_v4(dst + v * 16u, scale_round16<T>(reinterpret_cast<const uint4*>(src)[v], s));
    done = vecs * 16u / (uint32_t)sizeof(T);
  }
  for (uint32_t i = done + lane_id(); i < n; i += 32) {
    const uint32_t b = elem_bits(scale_round_to<T>(DT<T>::to_float(src[i]), s));
    if (sizeof(T) == 4)
      st_u32(dst + i * 4u, b);
    else
      st_u16(dst + i * 2u, (uint16_t)b);
  }
}

// Routed form: element e of a logical buffer of whole rows of p.row elements lives in row
// index[e / row] of `base`, column e % row (index == nullptr: the logical buffer is `base`). Called
// with the same e by every lane of a warp, so the index load is one broadcast. A row outside
// [0, rows) is never dereferenced: the status records which index held it and nullptr is returned.
template <typename T>
__device__ __forceinline__ T* a2a_row_addr(const A2aParams& p, T* base, const int64_t* index, uint64_t rows,
                                          uint32_t e, uint32_t which) {
  if (index == nullptr) return base + e;
  const uint32_t row = e / p.row;
  const int64_t i = index[row];
  if (i < 0 || (uint64_t)i >= rows) {
    if (lane_id() == 0) *p.status = (uint32_t)kSraBadIndex | ((uint32_t)p.rank << 8) | (which << 16);
    return nullptr;
  }
  return base + (uint64_t)i * p.row + (e - row * p.row);
}

// Combine: the warp has stored slot row s, columns [col, col + p.span) (docs/MEMORY_MODEL.md). Lane
// 0 sets bit s % topk of the segment's mask with acquire-release semantics; __syncwarp orders the
// lanes' stores before it and its acquire before their loads. A bit already set is a repeated slot
// (recorded; the segment then never fills). The warp that fills the mask writes the segment.
__device__ __forceinline__ uint32_t atom_or_acq_rel_gpu(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.acq_rel.gpu.global.or.b32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
template <typename T>
__device__ __forceinline__ void a2a_combine_arrive(const A2aParams& p, const T* dst) {
  const T* slots = reinterpret_cast<const T*>(p.out);
  const uint64_t e = (uint64_t)(dst - slots), H = p.row;
  const uint64_t s = e / H, t = s / p.topk;
  const uint32_t c = (uint32_t)(s - t * p.topk), seg = (uint32_t)(e - s * H) / p.span;
  __syncwarp();
  uint32_t old = 0;
  if (lane_id() == 0) old = atom_or_acq_rel_gpu(p.masks + t * (H / p.span) + seg, 1u << c);
  old = __shfl_sync(kAll, old, 0);
  if (old & (1u << c)) {
    if (lane_id() == 0) *p.status = (uint32_t)kSraBadIndex | ((uint32_t)p.rank << 8) | (2u << 16);
    return;
  }
  const uint32_t full = p.topk == 32u ? ~0u : (1u << p.topk) - 1u;
  if ((old | (1u << c)) != full) return;
  const uint64_t col = (uint64_t)seg * p.span;
  combine_segment<T>(slots + t * p.topk * H + col, H, p.gate + t * p.topk, p.topk,
                     reinterpret_cast<T*>(p.combine_out) + t * H + col, p.span);
}

// my own chunk, routed: one warp per row, through both indices (COMBINE: then arrives at every
// segment of the slot row; SCALE: the row's T(x * s), as sent to the peers)
template <typename T, bool COMBINE, bool SCALE = false>
__device__ __forceinline__ void a2a_copy_own_rows(const A2aParams& p) {
  const uint32_t H = p.row, rows = p.in_cnt[p.rank] / H;
  const uint32_t nwarps = gridDim.x * kSraWarps;
  for (uint32_t j = blockIdx.x * kSraWarps + (threadIdx.x >> 5); j < rows; j += nwarps) {
    const T* src = a2a_row_addr(p, reinterpret_cast<const T*>(p.in), p.in_index, p.in_rows, p.in_off[p.rank] + j * H, 0u);
    T* dst = a2a_row_addr(p, reinterpret_cast<T*>(p.out), p.out_index, p.out_rows, p.out_off[p.rank] + j * H, 1u);
    if (src == nullptr || dst == nullptr) continue;
    uint32_t done = 0;
    if constexpr (SCALE) {
      const float s = p.in_scale[p.in_off[p.rank] / H + j];
      if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0) {
        const uint32_t vecs = H * (uint32_t)sizeof(T) / 16u;
        for (uint32_t v = lane_id(); v < vecs; v += 32)
          reinterpret_cast<uint4*>(dst)[v] = scale_round16<T>(reinterpret_cast<const uint4*>(src)[v], s);
        done = vecs * 16u / (uint32_t)sizeof(T);
      }
      for (uint32_t i = done + lane_id(); i < H; i += 32) dst[i] = scale_round_to<T>(DT<T>::to_float(src[i]), s);
    } else {
      if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0) {
        const uint32_t vecs = H * (uint32_t)sizeof(T) / 16u;
        for (uint32_t v = lane_id(); v < vecs; v += 32)
          reinterpret_cast<uint4*>(dst)[v] = reinterpret_cast<const uint4*>(src)[v];
        done = vecs * 16u / (uint32_t)sizeof(T);
      }
      for (uint32_t i = done + lane_id(); i < H; i += 32) dst[i] = src[i];
    }
    if constexpr (COMBINE)
      for (uint32_t col = 0; col < H; col += p.span) a2a_combine_arrive<T>(p, dst + col);
  }
}

// my own chunk: a bit copy, spread over every thread of the grid
template <typename T>
__device__ __forceinline__ void a2a_copy_own(const A2aParams& p) {
  const uint64_t n = p.in_cnt[p.rank];
  if (n == 0) return;
  const T* src = reinterpret_cast<const T*>(p.in) + p.in_off[p.rank];
  T* dst = reinterpret_cast<T*>(p.out) + p.out_off[p.rank];
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (uint64_t)gridDim.x * blockDim.x;
  uint64_t done = 0;
  if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0) {
    const uint64_t vecs = n * sizeof(T) / 16u;
    for (uint64_t v = tid; v < vecs; v += nthr)
      reinterpret_cast<uint4*>(dst)[v] = reinterpret_cast<const uint4*>(src)[v];
    done = vecs * 16u / sizeof(T);
  }
  for (uint64_t i = done + tid; i < n; i += nthr) dst[i] = src[i];
}

// The items of window k of one pair on this lane: `m` blocks, block w of the window is chunk block
// lane + (k * bpw + w) * G; item t is item t % block_items of block t / block_items.
struct A2aWindow {
  uint32_t first_block;  // lane blocks k * bpw ..
  uint32_t m;            // blocks in this window
  uint32_t nitems;       // m * block_items (the chunk's last block may have fewer: skipped)
};
__device__ __forceinline__ A2aWindow a2a_window(const A2aGeom& g, uint32_t bpw, uint32_t k) {
  const uint32_t lb = a2a_lane_blocks(a2a_num_blocks(g), (int)blockIdx.x, (int)gridDim.x);
  A2aWindow w;
  w.first_block = k * bpw;
  w.m = min(bpw, lb - w.first_block);
  w.nitems = w.m * g.block_items;
  return w;
}
// item t of the window (false: past the chunk's last item); *wire = its block's offset in the lane's share
__device__ __forceinline__ bool a2a_window_item(const A2aGeom& g, const A2aWindow& w, uint32_t t, WarpItem& it,
                                                uint32_t& wire) {
  const uint32_t wb = t / g.block_items, j = t - wb * g.block_items;
  const uint32_t b = blockIdx.x + (w.first_block + wb) * gridDim.x;
  if (b + 1u == a2a_num_blocks(g) && j >= a2a_block_num_items(g, a2a_block_n(g, b))) return false;
  it = a2a_block_item(g, b, j);
  wire = wb * g.block_wire;
  return true;
}

// A full item of T(x * s) that is not vector aligned (SCALE): out of line, as full_send_unaligned
template <typename T, int KB, int GPL, int CODEC, typename DST>
__device__ __noinline__ void a2a_send_scaled_unaligned(const T* __restrict__ src, const WarpItem it, float s,
                                                       const RngKey rng, const DST ds) {
  float x[GPL][8];
  slice_load_scalar<T, GPL>(src, x);
  slice_scale_round<GPL, T>(x, s);
  if constexpr (CODEC != kMaxMin)
    full_send_fp8_x<CODEC, GPL>(x, it, rng, ds);
  else
    full_send_x<T, KB, GPL, false, false>(x, it, 1.0f, rng, ds, (T*)nullptr);
}

// one item of a chunk in an FP8 codec (KB 8 records; the SR codecs draw from the pair's key `rng`):
// to a peer's slot (OneDst), or to the codes output (CodesDst)
template <typename T, int CODEC, int GPL, typename DST>
__device__ __forceinline__ void a2a_send_item_fp8(const T* src, const WarpItem& it, const RngKey& rng,
                                                  const DST& push) {
  if (item_kind(it) == kItemFull) {
    if (group_aligned<T>(src)) {
      float x[GPL][8];
      slice_load_vec<T, GPL>(src, x);
      full_send_fp8_x<CODEC, GPL>(x, it, rng, push);
    } else {
      full_send_fp8_unaligned<T, CODEC, GPL>(src, it, rng, push);
    }
  } else {
    bucket_quantize_fp8<T, CODEC>(src, it, rng, push);
  }
}
// the same for the values T(x * s) (SCALE)
template <typename T, int CODEC, int GPL, typename DST>
__device__ __forceinline__ void a2a_send_item_fp8_scaled(const T* src, const WarpItem& it, const RngKey& rng,
                                                         const DST& push, float s) {
  if (item_kind(it) == kItemFull) {
    if (group_aligned<T>(src)) {
      float x[GPL][8];
      slice_load_vec<T, GPL>(src, x);
      slice_scale_round<GPL, T>(x, s);
      full_send_fp8_x<CODEC, GPL>(x, it, rng, push);
    } else {
      a2a_send_scaled_unaligned<T, 8, GPL, CODEC, DST>(src, it, s, rng, push);
    }
  } else {
    bucket_quantize_fp8_rounded<T, CODEC>(src, it, s, rng, push);
  }
}
template <typename T, int CODEC, int GPL>
__device__ __forceinline__ void a2a_recv_item_fp8(const uint8_t* rec, const WarpItem& it, T* dst) {
  if (item_kind(it) == kItemFull) {
    if (group_aligned<T>(dst)) {
      SliceWords<GPL> sw;
      slice_fetch<8, GPL>(rec, it.meta_off, it.pay_off, item_lpb_log2(it), 8, sw);
      full_recv_fp8_w<T, CODEC, GPL, true>(sw, dst);
    } else {
      full_recv_fp8_unaligned<T, CODEC, GPL>(rec, it, dst);
    }
  } else {
    bucket_recv_fp8<T, CODEC>(rec, it, dst);
  }
}

// one item of the values T(x * s) to a peer's slot (SCALE), every codec
template <typename T, int KB, int GPL, int CODEC>
__device__ __forceinline__ void a2a_send_item_scaled(const T* src, const WarpItem& it, float s, const RngKey& rng,
                                                     const OneDst& push) {
  if constexpr (CODEC != kMaxMin) {
    a2a_send_item_fp8_scaled<T, CODEC, GPL, OneDst>(src, it, rng, push, s);
    return;
  }
  const uint32_t kind = item_kind(it);
  if (kind == kItemFull) {
    if (group_aligned<T>(src)) {
      float x[GPL][8];
      slice_load_vec<T, GPL>(src, x);
      slice_scale_round<GPL, T>(x, s);
      full_send_x<T, KB, GPL, false, true>(x, it, 1.0f, rng, push, (T*)nullptr);
    } else {
      a2a_send_scaled_unaligned<T, KB, GPL, kMaxMin, OneDst>(src, it, s, rng, push);
    }
  } else if (kind == kItemBucket) {
    bucket_quantize_rounded<T, OneDst>(src, it, s, rng, push);
  } else {
    a2a_raw_send_scaled<T>(src, it, push.p, s);
  }
}

template <typename T, int KB, int GPL, bool IDX, int CODEC, bool SCALE>
__device__ __forceinline__ void a2a_send_window(const A2aParams& p, int q, uint32_t bpw, uint32_t k,
                                                const RngKey& rng) {
  const int r = p.rank;
  const A2aGeom g = a2a_geom(p.in_cnt[q], p.bits, p.bucket, (int)sizeof(T));
  const A2aWindow w = a2a_window(g, bpw, k);
  const T* chunk = reinterpret_cast<const T*>(p.in) + p.in_off[q];
  uint8_t* share = p.recv[q] + (size_t)r * p.slot_bytes + (size_t)blockIdx.x * p.lane_slot;
  const SrcSet no_src{nullptr, 0u, 0, -1};
  for (uint32_t t = threadIdx.x >> 5; t < w.nitems; t += kSraWarps) {
    WarpItem it;
    uint32_t wire;
    if (!a2a_window_item(g, w, t, it, wire)) continue;
    const OneDst push{share + wire};
    const T* src;
    if constexpr (IDX) {
      // the item lies inside one row (a2a_rows_fit): one index load moves all of it
      src = a2a_row_addr(p, reinterpret_cast<const T*>(p.in), p.in_index, p.in_rows, p.in_off[q] + it.elem_off, 0u);
      if (src == nullptr) continue;
    } else {
      src = chunk + it.elem_off;
    }
    if constexpr (SCALE) {
      // and one scale load
      a2a_send_item_scaled<T, KB, GPL, CODEC>(src, it, p.in_scale[(p.in_off[q] + it.elem_off) / p.row], rng, push);
      continue;
    }
    if constexpr (CODEC != kMaxMin) {
      a2a_send_item_fp8<T, CODEC, GPL, OneDst>(src, it, rng, push);
      continue;
    }
    const uint32_t kind = item_kind(it);
    if (kind == kItemFull) {
      if (group_aligned<T>(src)) {
        float x[GPL][8];
        slice_load_vec<T, GPL>(src, x);
        full_send_x<T, KB, GPL, false, true>(x, it, 1.0f, rng, push, (T*)nullptr);
      } else {
        full_send_unaligned<T, T, KB, GPL, false>(src, it, 1.0f, rng, push, (T*)nullptr);
      }
    } else if (kind == kItemBucket) {
      bucket_quantize<T, T>(src, it, 1.0f, rng, no_src, push, (T*)nullptr);
    } else {
      a2a_raw_send<T>(src, it, push.p);
    }
  }
}

// codes output: where element e of the logical receive buffer goes (p.out holds one code byte per
// element; nullptr: a bad index), and the scale of the bucket that starts there
__device__ __forceinline__ uint8_t* a2a_codes_addr(const A2aParams& p, bool idx, uint32_t e) {
  uint8_t* codes = reinterpret_cast<uint8_t*>(p.out);
  return idx ? a2a_row_addr(p, codes, p.out_index, p.out_rows, e, 1u) : codes + e;
}
__device__ __forceinline__ float* a2a_scales_addr(const A2aParams& p, const uint8_t* codes) {
  return p.out_scales + (uint64_t)(codes - reinterpret_cast<const uint8_t*>(p.out)) / p.bucket;
}

// codes output, my own chunk: every item through the peers' FP8 encoder, straight into (codes,
// scales), one warp per item over the whole grid; `rng` is the key of the pair (r, r)
template <typename T, int GPL, bool IDX, int CODEC>
__device__ __forceinline__ void a2a_encode_own(const A2aParams& p, const RngKey& rng) {
  const int r = p.rank;
  const A2aGeom g = a2a_geom(p.in_cnt[r], p.bits, p.bucket, (int)sizeof(T));
  const uint32_t nb = a2a_num_blocks(g), total = nb * g.block_items, nwarps = gridDim.x * kSraWarps;
  for (uint32_t t = blockIdx.x * kSraWarps + (threadIdx.x >> 5); t < total; t += nwarps) {
    const uint32_t b = t / g.block_items, j = t - b * g.block_items;
    if (b + 1u == nb && j >= a2a_block_num_items(g, a2a_block_n(g, b))) continue;
    const WarpItem it = a2a_block_item(g, b, j);
    const T* src;
    if constexpr (IDX) {
      src = a2a_row_addr(p, reinterpret_cast<const T*>(p.in), p.in_index, p.in_rows, p.in_off[r] + it.elem_off, 0u);
      if (src == nullptr) continue;
    } else {
      src = reinterpret_cast<const T*>(p.in) + p.in_off[r] + it.elem_off;
    }
    uint8_t* codes = a2a_codes_addr(p, IDX, p.out_off[r] + it.elem_off);
    if (codes == nullptr) continue;
    const CodesDst ds{codes, a2a_scales_addr(p, codes), it.meta_off, it.pay_off, item_n(it)};
    a2a_send_item_fp8<T, CODEC, GPL, CodesDst>(src, it, rng, ds);
  }
}

template <typename T, int KB, int GPL, bool IDX, int CODEC, bool CODES, bool COMBINE>
__device__ __forceinline__ void a2a_recv_window(const A2aParams& p, int q, uint32_t bpw, uint32_t k) {
  const int r = p.rank;
  const A2aGeom g = a2a_geom(p.out_cnt[q], p.bits, p.bucket, (int)sizeof(T));
  const A2aWindow w = a2a_window(g, bpw, k);
  T* chunk = reinterpret_cast<T*>(p.out) + p.out_off[q];
  const uint8_t* share = p.recv[r] + (size_t)q * p.slot_bytes + (size_t)blockIdx.x * p.lane_slot;
  for (uint32_t t = threadIdx.x >> 5; t < w.nitems; t += kSraWarps) {
    WarpItem it;
    uint32_t wire;
    if (!a2a_window_item(g, w, t, it, wire)) continue;
    const SrcSet ss{share + wire, 0u, 1, -1};
    if constexpr (CODES) {
      uint8_t* codes = a2a_codes_addr(p, IDX, p.out_off[q] + it.elem_off);
      if (codes != nullptr) fp8_unpack_item<GPL>(ss.base, it, codes, a2a_scales_addr(p, codes));
      continue;
    }
    T* dst;
    if constexpr (IDX) {
      dst = a2a_row_addr(p, reinterpret_cast<T*>(p.out), p.out_index, p.out_rows, p.out_off[q] + it.elem_off, 1u);
      if (dst == nullptr) continue;
    } else {
      dst = chunk + it.elem_off;
    }
    // COMBINE: the item is one span of one slot row (a2a_rows_fit)
    if constexpr (CODEC != kMaxMin) {
      a2a_recv_item_fp8<T, CODEC, GPL>(ss.base, it, dst);
      if constexpr (COMBINE) a2a_combine_arrive<T>(p, dst);
      continue;
    }
    const uint32_t kind = item_kind(it);
    if (kind == kItemFull) {
      if (group_aligned<T>(dst)) {
        SliceWords<GPL> sw;
        slice_fetch<KB, GPL>(ss.base, it.meta_off, it.pay_off, item_lpb_log2(it), KB ? KB : item_bits(it), sw);
        full_recv_w<T, KB, GPL, true>(sw, it, dst);
      } else {
        full_recv_unaligned<T, KB, GPL>(ss, it, dst);
      }
    } else if (kind == kItemBucket) {
      bucket_recv<T>(ss, it, dst);
    } else {
      raw_ag_recv<T>(ss, it, dst);
    }
    if constexpr (COMBINE) a2a_combine_arrive<T>(p, dst);
  }
}

// IDX: the routed form (A2aParams::in_index / out_index); only the item addresses and the own-chunk
// copy differ, and the plain instantiations compile as before.
// CODEC: the wire codec of the peers' chunks (quant_math.h); the FP8 ones exist with KB 8 only.
// CODES (FP8 codecs only, A2aParams::out_scales set): the output receives the codes and units of
// every chunk undecoded, the own chunk encoded like a peer's.
// COMBINE (routed, decoded output; A2aParams::combine_out set): the weighted top-k combine of the
// slots, finalized per segment by the last warp to store into it.
// SCALE (routed, decoded output, no combine; A2aParams::in_scale set): sent row i is T(x * in_scale[i]),
// the own rows included.
template <typename T, int KB, int GPL, bool IDX = false, int CODEC = kMaxMin, bool CODES = false, bool COMBINE = false,
          bool SCALE = false>
__global__ void __launch_bounds__(kSraThreads, kSraCtasPerSm) a2a_kernel(const __grid_constant__ A2aParams p) {
  static_assert(CODEC == kMaxMin || KB == 8, "the FP8 codecs use 8-bit records");
  static_assert(!CODES || CODEC != kMaxMin, "codes are delivered for the FP8 codecs only");
  static_assert(!COMBINE || (IDX && !CODES), "the combine needs the routed, decoded output");
  static_assert(!SCALE || (IDX && !CODES && !COMBINE), "the scaled send needs the routed, decoded output");
  __shared__ int s_abort;
  __shared__ uint32_t s_send[kMaxPeers], s_recv[kMaxPeers];  // this lane's windows per destination / source
  const int lane = blockIdx.x, r = p.rank, W = p.world;
  const uint32_t epoch = *reinterpret_cast<volatile uint32_t*>(&p.sync->epoch) + 1u;
  // every pair has the same window size: it depends on (slot, lanes, bits, bucket, dtype) only
  const uint32_t bpw = a2a_window_blocks(a2a_geom(0, p.bits, p.bucket, (int)sizeof(T)), p.lane_slot);
  if (threadIdx.x == 0) s_abort = 0;
  if (threadIdx.x < (uint32_t)kMaxPeers) {
    const int q = (int)threadIdx.x;
    const bool peer = q < W && q != r;
    s_send[q] = peer ? a2a_lane_windows(a2a_geom(p.in_cnt[q], p.bits, p.bucket, (int)sizeof(T)), lane, p.lanes, bpw) : 0u;
    s_recv[q] = peer ? a2a_lane_windows(a2a_geom(p.out_cnt[q], p.bits, p.bucket, (int)sizeof(T)), lane, p.lanes, bpw) : 0u;
  }
  __syncthreads();
  uint32_t rounds = 0;
  for (int q = 0; q < W; ++q) rounds = max(rounds, max(s_send[q], s_recv[q]));

  _Pragma("unroll 1") for (uint32_t k = 0; k < rounds; ++k) {
    const uint32_t wl = lane_id();
    const bool has_send = wl < (uint32_t)W && s_send[wl] > k, has_recv = wl < (uint32_t)W && s_recv[wl] > k;
    // 1. the destinations have released my previous window
    if (threadIdx.x < 32 && k > 0 &&
        !a2a_wait(p, p.released[r], has_send, a2a_tag(epoch, k - 1u), kSraTimeoutPhase2))
      s_abort = 1;
    __syncthreads();
    if (s_abort) break;
    // 2. push window k to every destination that has one, then announce it
    RngKey rng = p.rng;
    rng.seq += epoch - p.epoch_hint;  // graph replays advance the random stream
    for (int s = 1; s < W; ++s) {
      const int q = (r + s) % W;
      if (s_send[q] <= k) continue;
      rng.stream = a2a_rng_stream(p.rank_base + r, p.rank_base + q);
      a2a_send_window<T, KB, GPL, IDX, CODEC, SCALE>(p, q, bpw, k, rng);
    }
    __syncthreads();
    if (threadIdx.x < 32 && has_send)
      st_release_sys_u64(p.landed[wl] + (size_t)r * p.flag_stride + lane, a2a_tag(epoch, k));
    // 3. decode window k of every source that has one, then release it
    if (threadIdx.x < 32 && !a2a_wait(p, p.landed[r], has_recv, a2a_tag(epoch, k), kSraTimeoutPhase1)) s_abort = 1;
    __syncthreads();
    if (s_abort) break;
    for (int s = 1; s < W; ++s) {
      const int q = (r + W - s) % W;
      if (s_recv[q] > k) a2a_recv_window<T, KB, GPL, IDX, CODEC, CODES, COMBINE>(p, q, bpw, k);
    }
    __syncthreads();
    if (threadIdx.x < 32 && has_recv)
      st_release_sys_u64(p.released[wl] + (size_t)r * p.flag_stride + lane, a2a_tag(epoch, k));
  }

  // my own chunk last: the pushes to the peers are on the critical path, the copy is not
  if (!s_abort) {
    if constexpr (CODES) {
      RngKey rng = p.rng;
      rng.seq += epoch - p.epoch_hint;
      rng.stream = a2a_rng_stream(p.rank_base + r, p.rank_base + r);
      a2a_encode_own<T, GPL, IDX, CODEC>(p, rng);
    } else if constexpr (IDX) {
      a2a_copy_own_rows<T, COMBINE, SCALE>(p);
    } else {
      a2a_copy_own<T>(p);
    }
  }

  // slot handshake, as in rs_kernel: every lane, whether or not it had windows
  if (threadIdx.x < 32 && !s_abort) {
    const uint32_t flag = flag_value(epoch, 0), wl = lane_id();
    if (wl < (uint32_t)W && (int)wl != r) st_release_sys(p.flags2[wl] + (size_t)r * p.flag_stride + lane, flag);
    int rc = 0;
    if (wl < (uint32_t)W && (int)wl != r) {
      rc = wait_flag(p.flags2[r] + (size_t)wl * p.flag_stride + lane, flag, p.timeout_ns, p.abort_word);
      if (rc != 0) *p.status = (rc == 2 ? (uint32_t)kSraAborted : (uint32_t)kSraTimeoutPhase2) | (wl << 8) | ((uint32_t)lane << 16);
    }
    __syncwarp();
  }
  sync_finish(p.sync, epoch, p.lanes);
}

}  // namespace dev

// the combine instantiations: routed, decoded output, every codec and KB
template <typename T, int GPL>
cudaError_t launch_a2a_combine(const A2aParams& p, cudaStream_t stream) {
  if (p.out_scales != nullptr || (p.codec != kMaxMin && p.bits != 8)) return cudaErrorInvalidValue;
  if (p.codec != kMaxMin)
    return dispatch_fp8(p.codec, cudaErrorInvalidValue, [&](auto c) {
      dev::a2a_kernel<T, 8, GPL, true, decltype(c)::value, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p);
      return cudaGetLastError();
    });
  switch ((p.bits == 2 || p.bits == 4 || p.bits == 8) ? p.bits : 0) {
    case 2: dev::a2a_kernel<T, 2, GPL, true, kMaxMin, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    case 4: dev::a2a_kernel<T, 4, GPL, true, kMaxMin, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    case 8: dev::a2a_kernel<T, 8, GPL, true, kMaxMin, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    default: dev::a2a_kernel<T, 0, GPL, true, kMaxMin, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
  }
  return cudaGetLastError();
}

// the scaled-send instantiations: routed, decoded output, no combine, every codec and KB
template <typename T, int GPL>
cudaError_t launch_a2a_scaled(const A2aParams& p, cudaStream_t stream) {
  if (p.out_scales != nullptr || p.combine_out != nullptr || p.in_index == nullptr ||
      (p.codec != kMaxMin && p.bits != 8))
    return cudaErrorInvalidValue;
  if (p.codec != kMaxMin)
    return dispatch_fp8(p.codec, cudaErrorInvalidValue, [&](auto c) {
      dev::a2a_kernel<T, 8, GPL, true, decltype(c)::value, false, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p);
      return cudaGetLastError();
    });
  switch ((p.bits == 2 || p.bits == 4 || p.bits == 8) ? p.bits : 0) {
    case 2: dev::a2a_kernel<T, 2, GPL, true, kMaxMin, false, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    case 4: dev::a2a_kernel<T, 4, GPL, true, kMaxMin, false, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    case 8: dev::a2a_kernel<T, 8, GPL, true, kMaxMin, false, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    default: dev::a2a_kernel<T, 0, GPL, true, kMaxMin, false, false, true><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
  }
  return cudaGetLastError();
}

template <typename T, int GPL, bool IDX>
cudaError_t launch_a2a_gpl(const A2aParams& p, cudaStream_t stream) {
  if constexpr (IDX) {
    if (p.in_scale != nullptr) return launch_a2a_scaled<T, GPL>(p, stream);
    if (p.combine_out != nullptr) return launch_a2a_combine<T, GPL>(p, stream);
  }
  if (p.codec != kMaxMin) {
    if (p.bits != 8) return cudaErrorInvalidValue;
    const bool codes = p.out_scales != nullptr;
    return dispatch_fp8(p.codec, cudaErrorInvalidValue, [&](auto c) {
      if (codes)
        dev::a2a_kernel<T, 8, GPL, IDX, decltype(c)::value, true><<<p.lanes, kSraThreads, 0, stream>>>(p);
      else
        dev::a2a_kernel<T, 8, GPL, IDX, decltype(c)::value><<<p.lanes, kSraThreads, 0, stream>>>(p);
      return cudaGetLastError();
    });
  }
  if (p.out_scales != nullptr) return cudaErrorInvalidValue;
  const int kb = (p.bits == 2 || p.bits == 4 || p.bits == 8) ? p.bits : 0;
  switch (kb) {
    case 2: dev::a2a_kernel<T, 2, GPL, IDX><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    case 4: dev::a2a_kernel<T, 4, GPL, IDX><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    case 8: dev::a2a_kernel<T, 8, GPL, IDX><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
    default: dev::a2a_kernel<T, 0, GPL, IDX><<<p.lanes, kSraThreads, 0, stream>>>(p); break;
  }
  return cudaGetLastError();
}

template <typename T, bool IDX>
cudaError_t launch_a2a_idx(const A2aParams& p, cudaStream_t stream) {
  return a2a_slice_elems(p.bits, p.bucket) == 1024u ? launch_a2a_gpl<T, 4, IDX>(p, stream)
                                                    : launch_a2a_gpl<T, 2, IDX>(p, stream);
}

template <typename T>
cudaError_t launch_a2a_t(const A2aParams& p, cudaStream_t stream) {
  return (p.in_index != nullptr || p.out_index != nullptr) ? launch_a2a_idx<T, true>(p, stream)
                                                           : launch_a2a_idx<T, false>(p, stream);
}

}  // namespace cgx

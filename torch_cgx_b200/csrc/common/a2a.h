// Layout of one compressed all-to-all chunk, shared by the fused kernel, the host and the CPU
// simulator.
//
// An all-to-all call quantizes every chunk with ONE (bits, bucket) pair, so the blocks, warp items
// and record offsets of a chunk are a pure function of (elements, bits, bucket, dtype, slice size):
// exactly what build_plan makes of a one-layer table at element 0 with one chunk and one lane. The
// fused kernel derives them here on the device, so a call uploads no table whatever its splits,
// and sender and receiver agree on a pair's layout without exchanging anything.
//
// Windows. Lane c of a pair handles the chunk's blocks c, c + G, c + 2G, ... (G lanes) and streams
// them through its share of the receiver's slot for the sender, `bpw` blocks per window. Every full
// block has the same record size, so a window of `bpw` blocks always fits the lane's share; cuts
// fall on block boundaries, hence on bucket boundaries, and the quantized values do not depend on
// the slot size or the lane count.
#pragma once
#include <cstdint>
#include "wire.h"

namespace cgx {

struct A2aGeom {
  uint32_t n;            // elements of the chunk
  int bits;              // 1..8, or kRawBits
  uint32_t bucket;       // quantization bucket after the clamp to kMaxBlockElems (raw: kRawItemElems)
  uint32_t slice;        // elements of a kItemFull item: 1024 with 1024-element buckets, else 512
  int elsize;
  uint32_t block_elems;  // elements of a full block
  uint32_t block_wire;   // record bytes of a full block
  uint32_t block_items;  // warp items of a full block
};

// slice size of a call: build_plan's rule for a table whose only compressed layer has `bucket`
CGX_HD uint32_t a2a_slice_elems(int bits, uint32_t bucket) {
  return (bits < kRawBits && bucket == 1024u) ? 1024u : 512u;
}

// warp items of a block of n elements (build_plan's emit_items)
CGX_HD uint32_t a2a_block_num_items(const A2aGeom& g, uint32_t n) {
  if (g.bits >= kRawBits) return div_up(n, kRawItemElems);
  const uint32_t B = g.bucket;
  const bool pow2 = B >= 8u && (B & (B - 1u)) == 0u && B <= g.slice;
  if (!pow2) return div_up(n, B);
  const uint32_t full = n / g.slice;
  return full + div_up(n - full * g.slice, B);
}

CGX_HD A2aGeom a2a_geom(uint32_t n, int bits, uint32_t bucket, int elsize) {
  A2aGeom g;
  g.n = n;
  g.bits = bits >= kRawBits ? kRawBits : bits;
  uint32_t b = g.bits >= kRawBits ? kRawItemElems : bucket;
  b = b < 1u ? 1u : (b > kMaxBlockElems ? kMaxBlockElems : b);
  g.bucket = b;
  g.slice = a2a_slice_elems(g.bits, b);
  g.elsize = elsize;
  uint32_t per_block = kMaxBlockElems / b;
  per_block = per_block < 1u ? 1u : (per_block > kMaxBlockBuckets ? kMaxBlockBuckets : per_block);
  g.block_elems = per_block * b;
  g.block_wire = block_wire_bytes(g.block_elems, g.bits, b, elsize);
  g.block_items = a2a_block_num_items(g, g.block_elems);
  return g;
}

// (no n + block_elems - 1: a chunk may come within one block of 2^32 elements)
CGX_HD uint32_t a2a_num_blocks(const A2aGeom& g) { return g.n / g.block_elems + (g.n % g.block_elems ? 1u : 0u); }
CGX_HD uint32_t a2a_block_n(const A2aGeom& g, uint32_t b) {
  const uint32_t first = b * g.block_elems;
  return g.n - first < g.block_elems ? g.n - first : g.block_elems;
}

// record bytes of the whole chunk (its contiguous wire image)
CGX_HD uint64_t a2a_chunk_wire(const A2aGeom& g) {
  const uint32_t nb = a2a_num_blocks(g);
  if (nb == 0) return 0;
  return (uint64_t)(nb - 1u) * g.block_wire + block_wire_bytes(a2a_block_n(g, nb - 1u), g.bits, g.bucket, g.elsize);
}

// warp items of the whole chunk
CGX_HD uint32_t a2a_chunk_items(const A2aGeom& g) {
  const uint32_t nb = a2a_num_blocks(g);
  return nb == 0 ? 0u : (nb - 1u) * g.block_items + a2a_block_num_items(g, a2a_block_n(g, nb - 1u));
}

// Item j of block b. elem_off counts from the chunk's first element; meta_off / pay_off count from
// the block's record, which starts at b * block_wire in the chunk's contiguous wire image.
CGX_HD WarpItem a2a_block_item(const A2aGeom& g, uint32_t b, uint32_t j) {
  const uint32_t n = a2a_block_n(g, b);
  const uint32_t e0 = b * g.block_elems;
  WarpItem it;
  if (g.bits >= kRawBits) {
    const uint32_t off = j * kRawItemElems;
    const uint32_t cnt = n - off < kRawItemElems ? n - off : kRawItemElems;
    it.elem_off = e0 + off;
    it.meta_off = it.pay_off = off * (uint32_t)g.elsize;
    it.info = make_item_info(cnt == kRawItemElems ? kItemRaw : kItemRawTail, 0, kRawBits, cnt);
    return it;
  }
  const uint32_t B = g.bucket;
  const uint32_t mb = block_meta_bytes(n, B);
  const bool pow2 = B >= 8u && (B & (B - 1u)) == 0u && B <= g.slice;
  const uint32_t nfull = pow2 ? n / g.slice : 0u;
  if (j < nfull) {
    uint32_t lg = 0;
    while ((8u << lg) < B) ++lg;
    const uint32_t off = j * g.slice;
    it.elem_off = e0 + off;
    it.meta_off = (off / B) * 8u;
    it.pay_off = mb + (off / 8u) * (uint32_t)g.bits;
    it.info = make_item_info(kItemFull, lg, g.bits, g.slice);
    return it;
  }
  const uint32_t off = nfull * g.slice + (j - nfull) * B;
  const uint32_t cnt = n - off < B ? n - off : B;
  it.elem_off = e0 + off;
  it.meta_off = (off / B) * 8u;
  it.pay_off = mb + (off / B) * bucket_groups(B) * (uint32_t)g.bits;
  it.info = make_item_info(kItemBucket, 0, g.bits, cnt);
  return it;
}

// ---- routed rows --------------------------------------------------------------------------------
// The span of a routed item: every item a2a_block_item can produce for a chunk of whole rows of a
// multiple of this many elements lies inside one row and covers exactly this many elements. Items
// start at multiples of their span within a block, blocks at multiples of every span, and a chunk
// of rows ends on a row boundary; the span is 512 raw elements, the slice for power-of-two buckets
// up to the slice (a chunk of whole slices has no bucket tail), otherwise the clamped bucket. The
// element size does not enter.
CGX_HD uint32_t a2a_row_span(int bits, uint32_t bucket, int elsize) {
  const A2aGeom g = a2a_geom(0, bits, bucket, elsize);
  if (g.bits >= kRawBits) return kRawItemElems;
  if (g.bucket >= 8u && (g.bucket & (g.bucket - 1u)) == 0u && g.bucket <= g.slice) return g.slice;
  return g.bucket;
}
// True iff the routed kernel can address every item of a chunk of whole rows of H elements as one
// span of one indexed row: H is a multiple of the span.
CGX_HD bool a2a_rows_fit(uint32_t H, int bits, uint32_t bucket, int elsize) {
  return H >= 1u && H % a2a_row_span(bits, bucket, elsize) == 0u;
}

// ---- windows ----------------------------------------------------------------------------------
// a lane's share of a per-source slot (16-byte granular)
CGX_HD uint32_t a2a_lane_slot_bytes(uint32_t slot_bytes, int lanes) {
  return slot_bytes / (uint32_t)lanes / kWireAlign * kWireAlign;
}
// blocks of one window (0: a full block does not fit the lane's share)
CGX_HD uint32_t a2a_window_blocks(const A2aGeom& g, uint32_t lane_slot) { return lane_slot / g.block_wire; }
// blocks of the chunk handled by `lane`: lane, lane + lanes, ...
CGX_HD uint32_t a2a_lane_blocks(uint32_t nblocks, int lane, int lanes) {
  return nblocks > (uint32_t)lane ? (nblocks - (uint32_t)lane - 1u) / (uint32_t)lanes + 1u : 0u;
}
CGX_HD uint32_t a2a_lane_windows(const A2aGeom& g, int lane, int lanes, uint32_t bpw) {
  return div_up(a2a_lane_blocks(a2a_num_blocks(g), lane, lanes), bpw);
}

// Largest world of an all-to-all: a2a_rng_stream keeps every pair of ranks below it apart.
constexpr int kA2aMaxWorld = 256;

// Random stream of the chunk world rank `src` sends to world rank `dst`: every pair has its own,
// and the counters are the chunk's element indices. The low parts of the ranks (mod 16) give the
// stream word's bits 0..8, exactly 2 * (src * 16 + dst) below 16 ranks; the high parts (src / 16,
// dst / 16, four bits each) go to bits 9..16. rounding_bits multiplies the word by an odd constant
// into the Philox key, a bijection, so distinct words are distinct keys.
CGX_HD uint32_t a2a_rng_stream(int src, int dst) {
  const uint32_t s = (uint32_t)src, d = (uint32_t)dst, P = (uint32_t)kMaxPeers;
  return 2u * ((s % P) * P + d % P) | (((s / P) | (d / P) << 4) << 9);
}

// Bytes of a chunk's region in the send or receive buffer of the cross-node all-to-all (and of
// Reducer::all_to_all): its records, rounded up to 256 so every region starts 256-byte aligned.
CGX_HD uint64_t a2a_region_bytes(uint64_t wire) { return (wire + 255u) / 256u * 256u; }

}  // namespace cgx

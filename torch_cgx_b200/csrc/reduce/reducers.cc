#include "reducers.h"

#include <algorithm>
#include <stdexcept>

#include "../common/a2a.h"
#include "fused_sra.h"  // shard_elems, replicate, check_all_to_all

namespace cgx {
namespace {

// Blocks [first, first + count) of `p` in maximal runs of compressed or of raw blocks, each with
// the codec it travels in: an FP8 codec covers the compressed blocks, raw blocks are raw either way.
template <class F>
void codec_runs(const Plan& p, uint32_t first, uint32_t count, WireCodec codec, F&& f) {
  if (codec == kMaxMin) {
    f(first, count, kMaxMin);
    return;
  }
  for (uint32_t b = first, end = first + count; b < end;) {
    const bool raw = block_bits(p.blocks[b]) >= kRawBits;
    uint32_t e = b + 1;
    while (e < end && (block_bits(p.blocks[e]) >= kRawBits) == raw) ++e;
    f(b, e - b, raw ? kMaxMin : codec);
    b = e;
  }
}

}  // namespace

Reducer::Reducer(Communicator* comm, BlockBackend* ops) : comm_(comm), ops_(ops) {}

Reducer::~Reducer() {
  for (Buf& b : bufs_)
    if (b.p) ops_->release(b.p);
}

const DevicePlan& Reducer::plan_for(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                                    cudaStream_t stream, int world) {
  PlanOptions opt;
  opt.world = world > 0 ? world : comm_->size();
  opt.lanes = 1;  // rank chunks only: one kernel launch per chunk handles all of its blocks
  opt.dtype = dtype;
  opt.skip_incomplete = skip_incomplete;
  const DevicePlan& dp = plans_.get(layers, opt, stream);
  if (ops_->is_cuda()) plans_.upload(dp, stream);
  return dp;
}

uint8_t* Reducer::scratch(int slot, size_t bytes) {
  if ((int)bufs_.size() <= slot) bufs_.resize(slot + 1);
  Buf& b = bufs_[slot];
  if (b.cap < bytes) {
    if (b.p) ops_->release(b.p);
    b.cap = std::max(bytes, b.cap * 2);
    b.p = static_cast<uint8_t*>(ops_->alloc(b.cap));
  }
  return b.p;
}

void Reducer::chunk_span(const Plan& p, int chunk, uint32_t* lo, uint32_t* hi) {
  uint32_t a = ~0u, b = 0;
  const uint32_t first = chunk < 0 ? 0 : p.chunk_begin(chunk);
  const uint32_t last = chunk < 0 ? (uint32_t)p.blocks.size() : p.chunk_end(chunk);
  for (uint32_t i = first; i < last; ++i) {
    a = std::min(a, p.blocks[i].elem_off);
    b = std::max(b, p.blocks[i].elem_off + block_n(p.blocks[i]));
  }
  if (a == ~0u) a = b = 0;
  *lo = a;
  *hi = b;
}

void Reducer::broadcast(void* data, size_t bytes, int root, cudaStream_t stream) {
  const int W = comm_->size(), r = comm_->rank();
  if (W == 1 || bytes == 0) return;
  std::vector<P2POp> ops;
  if (r == root) {
    for (int p = 0; p < W; ++p)
      if (p != root) ops.push_back({true, data, bytes, p});
    bytes_sent_ += bytes * (uint64_t)(W - 1);
  } else {
    ops.push_back({false, data, bytes, root});
  }
  comm_->exchange(ops, stream);
}

void Reducer::broadcast_compressed(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete,
                                   int root, const RngParams& rng, cudaStream_t stream, WireCodec codec) {
  const int W = comm_->size(), r = comm_->rank();
  if (W == 1) return;
  const DevicePlan& dp = plan_for(layers, dtype, skip_incomplete, stream, 1);  // the whole buffer is one chunk
  const Plan& plan = dp.plan;
  if (plan.blocks.empty()) return;
  const uint32_t nb = (uint32_t)plan.blocks.size();
  const size_t bytes = plan.chunk_wire_bytes[0];
  uint8_t* wire = scratch(4, row_bytes(plan));
  std::vector<P2POp> x;
  if (r == root) {
    // the root keeps what the receivers will decode
    codec_runs(plan, 0, nb, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
      ops_->quantize(dp, data, b, n, wire, 1.0f, make_rng_key(rng, root, 2), stream, c);
      ops_->dequantize(dp, wire, b, n, data, stream, c);
    });
    for (int p = 0; p < W; ++p)
      if (p != root) x.push_back({true, wire, bytes, p});
    bytes_sent_ += bytes * (uint64_t)(W - 1);
    comm_->exchange(x, stream);
  } else {
    x.push_back({false, wire, bytes, root});
    comm_->exchange(x, stream);
    codec_runs(plan, 0, nb, codec,
               [&](uint32_t b, uint32_t n, WireCodec c) { ops_->dequantize(dp, wire, b, n, data, stream, c); });
  }
}

// ------------------------------------------------------- sharded collectives --
void Reducer::reduce_scatter(const void* in, void* out, int dtype, const std::vector<LayerSpec>& shard_layers,
                             bool skip_incomplete, float prescale, const RngParams& rng, cudaStream_t stream,
                             WireCodec codec) {
  const int W = comm_->size(), r = comm_->rank();
  const uint64_t S = shard_elems(shard_layers);
  if (S == 0) return;
  if (S * (uint64_t)W >= (1ull << 32))
    throw std::invalid_argument("cgx reduce_scatter: the input exceeds 2^32 elements");
  const DevicePlan& dp = plan_for(replicate(shard_layers, W, S), dtype, skip_incomplete, stream);
  const Plan& plan = dp.plan;
  const size_t row = row_bytes(plan);
  uint8_t* sendb = scratch(0, row * W);
  uint8_t* recvb = scratch(1, row * W);
  uint32_t lo, hi;
  chunk_span(plan, r, &lo, &hi);
  float* acc = reinterpret_cast<float*>(scratch(3, (size_t)(hi - lo) * sizeof(float) + 16));
  const uint32_t cb = plan.chunk_begin(r), cn = plan.chunk_end(r) - cb;
  // my quantized copy of every peer's chunk -> that peer (the SRA's phase 1)
  std::vector<P2POp> x;
  for (int p = 0; p < W; ++p) {
    if (p == r) continue;
    const uint32_t pb = plan.chunk_begin(p), pn = plan.chunk_end(p) - pb;
    codec_runs(plan, pb, pn, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
      ops_->quantize(dp, in, b, n, sendb + row * p, prescale, make_rng_key(rng, r, 0), stream, c);
    });
    if (plan.chunk_wire_bytes[p]) x.push_back({true, sendb + row * p, plan.chunk_wire_bytes[p], p});
    if (plan.chunk_wire_bytes[r]) x.push_back({false, recvb + row * p, plan.chunk_wire_bytes[r], p});
    bytes_sent_ += plan.chunk_wire_bytes[p];
  }
  comm_->exchange(x, stream);
  if (!cn) return;
  ops_->accumulate(dp, nullptr, cb, cn, acc, lo, in, prescale, stream);
  for (int q = 0; q < W; ++q)
    if (q != r)
      codec_runs(plan, cb, cn, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
        ops_->accumulate(dp, recvb + row * q, b, n, acc, lo, nullptr, 1.0f, stream, c);
      });
  // store the fp32 sums as T: a raw plan of one shard does exactly that (acc[i] is element i of the
  // shard, chunk r starting at r * S)
  std::vector<LayerSpec> raw = shard_layers;
  for (LayerSpec& l : raw) l.bits = kRawBits;
  const DevicePlan& rp = plan_for(raw, dtype, false, stream, 1);
  ops_->quantize_f32(rp, acc, lo - (uint32_t)(r * S), 0, (uint32_t)rp.plan.blocks.size(),
                     scratch(2, row_bytes(rp.plan)), make_rng_key(rng, r, 1), out, stream);
}

void Reducer::all_gather(const void* in, void* out, int dtype, const std::vector<LayerSpec>& shard_layers,
                         bool skip_incomplete, const RngParams& rng, cudaStream_t stream, WireCodec codec,
                         float* out_scales) {
  const int W = comm_->size(), r = comm_->rank();
  const uint64_t S = shard_elems(shard_layers);
  if (out_scales != nullptr) check_sharded_buffers(ShardedOp::kAllGather, shard_layers, dtype, in, out, S, r, W, codec,
                                                   out_scales);
  if (S == 0) return;
  if (S * (uint64_t)W >= (1ull << 32))
    throw std::invalid_argument("cgx all_gather: the output exceeds 2^32 elements");
  const DevicePlan& dp = plan_for(replicate(shard_layers, W, S), dtype, skip_incomplete, stream);
  const Plan& plan = dp.plan;
  const size_t row = row_bytes(plan);
  uint8_t* recvb = scratch(1, row * W);
  uint8_t* mine = scratch(2, row);
  const size_t shard_bytes = (size_t)S * dtype_size(dtype);
  uint8_t* codes = static_cast<uint8_t*>(out);
  const uint32_t cb = plan.chunk_begin(r), cn = plan.chunk_end(r) - cb;
  if (out_scales != nullptr) {
    // the plan addresses my shard at element r * S of the output: read it from `in` through a base
    // shifted by that much, quantize it once and hand over the record the peers receive
    const uint8_t* base = static_cast<const uint8_t*>(in) - (size_t)r * shard_bytes;
    ops_->quantize(dp, base, cb, cn, mine, 1.0f, make_rng_key(rng, r, 1), stream, codec);
    ops_->unpack_fp8(dp, mine, cb, cn, codes, out_scales, stream);
  } else {
    uint8_t* own = static_cast<uint8_t*>(out) + (size_t)r * shard_bytes;
    if (in != own) ops_->copy(own, in, shard_bytes, stream);
    // the root's part of the compressed broadcast: quantize once, keep what the peers will decode
    codec_runs(plan, cb, cn, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
      ops_->quantize(dp, out, b, n, mine, 1.0f, make_rng_key(rng, r, 1), stream, c);
      ops_->dequantize(dp, mine, b, n, out, stream, c);
    });
  }
  std::vector<P2POp> x;
  for (int p = 0; p < W; ++p) {
    if (p == r) continue;
    if (plan.chunk_wire_bytes[r]) x.push_back({true, mine, plan.chunk_wire_bytes[r], p});
    if (plan.chunk_wire_bytes[p]) x.push_back({false, recvb + row * p, plan.chunk_wire_bytes[p], p});
    bytes_sent_ += plan.chunk_wire_bytes[r];
  }
  comm_->exchange(x, stream);
  for (int p = 0; p < W; ++p) {
    if (p == r) continue;
    const uint32_t pb = plan.chunk_begin(p), pn = plan.chunk_end(p) - pb;
    if (out_scales != nullptr) {
      ops_->unpack_fp8(dp, recvb + row * p, pb, pn, codes, out_scales, stream);
      continue;
    }
    codec_runs(plan, pb, pn, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
      ops_->dequantize(dp, recvb + row * p, b, n, out, stream, c);
    });
  }
}

void Reducer::all_to_all(const void* in, void* out, const std::vector<uint64_t>& in_counts,
                         const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec,
                         uint32_t bucket, const RngParams& rng, cudaStream_t stream, float* out_scales,
                         int rank_base) {
  const int W = comm_->size(), r = comm_->rank();
  check_all_to_all(in, out, in_counts, out_counts, dtype, bits, codec, bucket, r, W, nullptr, out_scales);
  if (out_scales != nullptr) {
    all_to_all_codes(in, static_cast<uint8_t*>(out), out_scales, in_counts, out_counts, dtype, codec, bucket, rng, stream,
                     rank_base);
    return;
  }
  const size_t es = (size_t)dtype_size(dtype);
  const bool raw = bits >= kRawBits;
  const uint8_t* src = static_cast<const uint8_t*>(in);
  uint8_t* dst = static_cast<uint8_t*>(out);
  // A peer chunk's record bytes follow from its size (common/a2a.h, which is build_plan's one-layer
  // plan of the chunk); its plan is asked for right where it is quantized or decoded.
  std::vector<size_t> io(W), oo(W), sw(W, 0), rw(W, 0), so(W + 1, 0), ro(W + 1, 0);
  uint64_t i = 0, o = 0;
  for (int q = 0; q < W; ++q) {
    io[q] = (size_t)i * es;
    oo[q] = (size_t)o * es;
    i += in_counts[q];
    o += out_counts[q];
    if (q != r && !raw) {
      sw[q] = a2a_chunk_wire(a2a_geom((uint32_t)in_counts[q], bits, bucket, (int)es));
      rw[q] = a2a_chunk_wire(a2a_geom((uint32_t)out_counts[q], bits, bucket, (int)es));
    }
    so[q + 1] = so[q] + a2a_region_bytes(sw[q]);
    ro[q + 1] = ro[q] + a2a_region_bytes(rw[q]);
  }
  if (in_counts[r]) ops_->copy(dst + oo[r], src + io[r], in_counts[r] * es, stream);
  uint8_t* sendb = raw ? nullptr : scratch(0, so[W] + 16);
  uint8_t* recvb = raw ? nullptr : scratch(1, ro[W] + 16);
  for (int q = 0; q < W; ++q) {
    if (!sw[q]) continue;
    RngKey key = make_rng_key(rng, r, 0);
    key.stream = a2a_rng_stream(rank_base + r, rank_base + q);
    const DevicePlan& dp = plan_for({LayerSpec{0, in_counts[q], bits, bucket}}, dtype, false, stream, 1);
    ops_->quantize(dp, src + io[q], 0, (uint32_t)dp.plan.blocks.size(), sendb + so[q], 1.0f, key, stream, codec);
  }
  std::vector<P2POp> x;
  for (int q = 0; q < W; ++q) {
    if (q == r) continue;
    if (raw) {
      if (in_counts[q]) x.push_back({true, const_cast<uint8_t*>(src + io[q]), in_counts[q] * es, q});
      if (out_counts[q]) x.push_back({false, dst + oo[q], out_counts[q] * es, q});
      bytes_sent_ += in_counts[q] * es;
      continue;
    }
    if (sw[q]) x.push_back({true, sendb + so[q], sw[q], q});
    if (rw[q]) x.push_back({false, recvb + ro[q], rw[q], q});
    bytes_sent_ += sw[q];
  }
  comm_->exchange(x, stream);
  for (int q = 0; q < W; ++q) {
    if (!rw[q]) continue;
    const DevicePlan& dp = plan_for({LayerSpec{0, out_counts[q], bits, bucket}}, dtype, false, stream, 1);
    ops_->dequantize(dp, recvb + ro[q], 0, (uint32_t)dp.plan.blocks.size(), dst + oo[q], stream, codec);
  }
}

void Reducer::all_to_all_codes(const void* in, uint8_t* codes, float* scales, const std::vector<uint64_t>& in_counts,
                               const std::vector<uint64_t>& out_counts, int dtype, WireCodec codec, uint32_t bucket,
                               const RngParams& rng, cudaStream_t stream, int rank_base) {
  const int W = comm_->size(), r = comm_->rank();
  const size_t es = (size_t)dtype_size(dtype);
  const uint8_t* src = static_cast<const uint8_t*>(in);
  // every chunk has a record here, the own one included; element offsets of the outputs
  std::vector<size_t> io(W), oo(W), sw(W), rw(W), so(W + 1, 0), ro(W + 1, 0);
  uint64_t i = 0, o = 0;
  for (int q = 0; q < W; ++q) {
    io[q] = (size_t)i * es;
    oo[q] = (size_t)o;
    i += in_counts[q];
    o += out_counts[q];
    sw[q] = a2a_chunk_wire(a2a_geom((uint32_t)in_counts[q], 8, bucket, (int)es));
    rw[q] = q == r ? 0 : a2a_chunk_wire(a2a_geom((uint32_t)out_counts[q], 8, bucket, (int)es));
    so[q + 1] = so[q] + (sw[q] + 255) / 256 * 256;
    ro[q + 1] = ro[q] + (rw[q] + 255) / 256 * 256;
  }
  uint8_t* sendb = scratch(0, so[W] + 16);
  uint8_t* recvb = scratch(1, ro[W] + 16);
  for (int q = 0; q < W; ++q) {
    if (!sw[q]) continue;
    RngKey key = make_rng_key(rng, r, 0);
    key.stream = a2a_rng_stream(rank_base + r, rank_base + q);
    const DevicePlan& dp = plan_for({LayerSpec{0, in_counts[q], 8, bucket}}, dtype, false, stream, 1);
    ops_->quantize(dp, src + io[q], 0, (uint32_t)dp.plan.blocks.size(), sendb + so[q], 1.0f, key, stream, codec);
    if (q == r) ops_->unpack_fp8(dp, sendb + so[q], 0, (uint32_t)dp.plan.blocks.size(), codes + oo[r], scales + oo[r] / bucket, stream);
  }
  std::vector<P2POp> x;
  for (int q = 0; q < W; ++q) {
    if (q == r) continue;
    if (sw[q]) x.push_back({true, sendb + so[q], sw[q], q});
    if (rw[q]) x.push_back({false, recvb + ro[q], rw[q], q});
    bytes_sent_ += sw[q];
  }
  comm_->exchange(x, stream);
  for (int q = 0; q < W; ++q) {
    if (!rw[q]) continue;
    const DevicePlan& dp = plan_for({LayerSpec{0, out_counts[q], 8, bucket}}, dtype, false, stream, 1);
    ops_->unpack_fp8(dp, recvb + ro[q], 0, (uint32_t)dp.plan.blocks.size(), codes + oo[q], scales + oo[q] / bucket, stream);
  }
}

// ---------------------------------------------------------------------- SRA --
void SraReducer::allreduce(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete,
                           float prescale, const RngParams& rng, cudaStream_t stream, WireCodec codec) {
  const DevicePlan& dp = plan_for(layers, dtype, skip_incomplete, stream);
  const Plan& plan = dp.plan;
  if (plan.blocks.empty()) return;
  const int W = comm_->size(), r = comm_->rank();
  const size_t row = row_bytes(plan);
  uint8_t* sendb = scratch(0, row * W);
  uint8_t* recvb = scratch(1, row * W);
  uint8_t* mine = scratch(2, row);
  uint32_t lo, hi;
  chunk_span(plan, r, &lo, &hi);
  float* acc = reinterpret_cast<float*>(scratch(3, (size_t)(hi - lo) * sizeof(float) + 16));
  const uint32_t cb = plan.chunk_begin(r), cn = plan.chunk_end(r) - cb;

  // phase 1: my quantized copy of every peer's chunk -> that peer
  std::vector<P2POp> x;
  for (int p = 0; p < W; ++p) {
    if (p == r) continue;
    const uint32_t pb = plan.chunk_begin(p), pn = plan.chunk_end(p) - pb;
    if (pn)
      codec_runs(plan, pb, pn, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
        ops_->quantize(dp, data, b, n, sendb + row * p, prescale, make_rng_key(rng, r, 0), stream, c);
      });
    if (plan.chunk_wire_bytes[p]) x.push_back({true, sendb + row * p, plan.chunk_wire_bytes[p], p});
    if (plan.chunk_wire_bytes[r]) x.push_back({false, recvb + row * p, plan.chunk_wire_bytes[r], p});
    bytes_sent_ += plan.chunk_wire_bytes[p];
  }
  comm_->exchange(x, stream);
  // reduce my chunk in fp32: own raw values first, then the peers in rank order
  if (cn) {
    ops_->accumulate(dp, nullptr, cb, cn, acc, lo, data, prescale, stream);
    for (int q = 0; q < W; ++q)
      if (q != r)
        codec_runs(plan, cb, cn, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
          ops_->accumulate(dp, recvb + row * q, b, n, acc, lo, nullptr, 1.0f, stream, c);
        });
    // requantize + self-decode so that every rank ends with identical values
    codec_runs(plan, cb, cn, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
      ops_->quantize_f32(dp, acc, lo, b, n, mine, make_rng_key(rng, r, 1), data, stream, c);
    });
  }
  // phase 2: all-gather of the reduced chunks
  x.clear();
  for (int p = 0; p < W; ++p) {
    if (p == r) continue;
    if (plan.chunk_wire_bytes[r]) x.push_back({true, mine, plan.chunk_wire_bytes[r], p});
    if (plan.chunk_wire_bytes[p]) x.push_back({false, recvb + row * p, plan.chunk_wire_bytes[p], p});
    bytes_sent_ += plan.chunk_wire_bytes[r];
  }
  comm_->exchange(x, stream);
  for (int p = 0; p < W; ++p) {
    if (p == r) continue;
    const uint32_t pb = plan.chunk_begin(p), pn = plan.chunk_end(p) - pb;
    if (pn)
      codec_runs(plan, pb, pn, codec, [&](uint32_t b, uint32_t n, WireCodec c) {
        ops_->dequantize(dp, recvb + row * p, b, n, data, stream, c);
      });
  }
}

// --------------------------------------------------------------------- Ring --
void RingReducer::allreduce(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete,
                            float prescale, const RngParams& rng, cudaStream_t stream, WireCodec codec) {
  const DevicePlan& dp = plan_for(layers, dtype, skip_incomplete, stream);
  const Plan& plan = dp.plan;
  if (plan.blocks.empty()) return;
  const int W = comm_->size(), r = comm_->rank();
  const size_t row = row_bytes(plan);
  uint8_t* bufa = scratch(0, row);
  uint8_t* bufb = scratch(1, row);
  uint32_t lo, hi;
  chunk_span(plan, -1, &lo, &hi);
  float* acc = reinterpret_cast<float*>(scratch(3, (size_t)(hi - lo) * sizeof(float) + 16));
  const uint32_t nblocks = (uint32_t)plan.blocks.size();
  auto cb = [&](int c) { return plan.chunk_begin(c); };
  auto cn = [&](int c) { return plan.chunk_end(c) - plan.chunk_begin(c); };
  ops_->accumulate(dp, nullptr, 0, nblocks, acc, lo, data, prescale, stream);
  const int right = (r + 1) % W, left = (r + W - 1) % W;
  // reduce-scatter: W-1 hops, the travelling partial sum is requantized at every hop
  for (int s = 0; s + 1 < W; ++s) {
    const int sseg = (r - s + W) % W, rseg = (r - s - 1 + 2 * W) % W;
    RngParams hop = rng;
    hop.seq = rng.seq * 16u + (uint32_t)s;
    if (cn(sseg))
      codec_runs(plan, cb(sseg), cn(sseg), codec, [&](uint32_t b, uint32_t n, WireCodec c) {
        ops_->quantize_f32(dp, acc, lo, b, n, bufa, make_rng_key(hop, r, 0), nullptr, stream, c);
      });
    std::vector<P2POp> x;
    if (plan.chunk_wire_bytes[sseg]) x.push_back({true, bufa, plan.chunk_wire_bytes[sseg], right});
    if (plan.chunk_wire_bytes[rseg]) x.push_back({false, bufb, plan.chunk_wire_bytes[rseg], left});
    bytes_sent_ += plan.chunk_wire_bytes[sseg];
    comm_->exchange(x, stream);
    if (cn(rseg))
      codec_runs(plan, cb(rseg), cn(rseg), codec, [&](uint32_t b, uint32_t n, WireCodec c) {
        ops_->accumulate(dp, bufb, b, n, acc, lo, nullptr, 1.0f, stream, c);
      });
  }
  // the fully reduced segment of this rank: requantize once more and self-decode
  int cur = (r + 1) % W;
  if (W == 1) cur = 0;
  RngParams fin = rng;
  fin.seq = rng.seq * 16u + 15u;
  uint8_t* have = bufa;
  uint8_t* next = bufb;
  if (cn(cur))
    codec_runs(plan, cb(cur), cn(cur), codec, [&](uint32_t b, uint32_t n, WireCodec c) {
      ops_->quantize_f32(dp, acc, lo, b, n, have, make_rng_key(fin, r, 1), data, stream, c);
    });
  // all-gather: forward the already-compressed bytes around the ring, decode locally
  for (int s = 0; s + 1 < W; ++s) {
    const int rseg = (cur + W - 1) % W;
    std::vector<P2POp> x;
    if (plan.chunk_wire_bytes[cur]) x.push_back({true, have, plan.chunk_wire_bytes[cur], right});
    if (plan.chunk_wire_bytes[rseg]) x.push_back({false, next, plan.chunk_wire_bytes[rseg], left});
    bytes_sent_ += plan.chunk_wire_bytes[cur];
    comm_->exchange(x, stream);
    if (cn(rseg))
      codec_runs(plan, cb(rseg), cn(rseg), codec, [&](uint32_t b, uint32_t n, WireCodec c) {
        ops_->dequantize(dp, next, b, n, data, stream, c);
      });
    std::swap(have, next);
    cur = rseg;
  }
}

// ----------------------------------------------------------------- AllToAll --
void AllToAllReducer::allreduce(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete,
                                float prescale, const RngParams& rng, cudaStream_t stream, WireCodec codec) {
  if (codec != kMaxMin) throw std::invalid_argument(kAllToAllNoFp8);
  const DevicePlan& dp = plan_for(layers, dtype, skip_incomplete, stream);
  const Plan& plan = dp.plan;
  if (plan.blocks.empty()) return;
  const int W = comm_->size(), r = comm_->rank();
  const size_t row = row_bytes(plan);
  const size_t whole = row * W;  // chunk c of the wire image lives at row * c
  uint8_t* sendb = scratch(0, whole);
  uint8_t* recvb = scratch(1, whole * W);
  uint32_t lo, hi;
  chunk_span(plan, -1, &lo, &hi);
  float* acc = reinterpret_cast<float*>(scratch(3, (size_t)(hi - lo) * sizeof(float) + 16));
  for (int c = 0; c < W; ++c) {
    const uint32_t b0 = plan.chunk_begin(c), bn = plan.chunk_end(c) - b0;
    if (bn) ops_->quantize(dp, data, b0, bn, sendb + row * c, prescale, make_rng_key(rng, r, 0), stream);
  }
  std::vector<P2POp> x;
  for (int p = 0; p < W; ++p) {
    if (p == r) continue;
    x.push_back({true, sendb, whole, p});
    x.push_back({false, recvb + whole * p, whole, p});
    bytes_sent_ += whole;
  }
  comm_->exchange(x, stream);
  ops_->accumulate(dp, nullptr, 0, (uint32_t)plan.blocks.size(), acc, lo, data, prescale, stream);
  for (int q = 0; q < W; ++q) {
    if (q == r) continue;
    for (int c = 0; c < W; ++c) {
      const uint32_t b0 = plan.chunk_begin(c), bn = plan.chunk_end(c) - b0;
      if (bn) ops_->accumulate(dp, recvb + whole * q + row * c, b0, bn, acc, lo, nullptr, 1.0f, stream);
    }
  }
  // store the fp32 sums back as T: a "raw" plan of the same layers does exactly that
  std::vector<LayerSpec> raw = layers;
  for (LayerSpec& l : raw) l.bits = kRawBits;
  const DevicePlan& rdp = plan_for(raw, dtype, false, stream);
  const Plan& rp = rdp.plan;
  uint8_t* tmp = scratch(2, row_bytes(rp) * W);
  for (int c = 0; c < W; ++c) {
    const uint32_t b0 = rp.chunk_begin(c), bn = rp.chunk_end(c) - b0;
    if (bn) ops_->quantize_f32(rdp, acc, lo, b0, bn, tmp + row_bytes(rp) * c, make_rng_key(rng, r, 1), data, stream);
  }
}

std::unique_ptr<Reducer> make_reducer(ReductionType type, Communicator* comm, BlockBackend* ops) {
  switch (type) {
    case ReductionType::kRing: return std::make_unique<RingReducer>(comm, ops);
    case ReductionType::kAllToAll: return std::make_unique<AllToAllReducer>(comm, ops);
    default: return std::make_unique<SraReducer>(comm, ops);
  }
}

}  // namespace cgx

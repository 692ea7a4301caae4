#include "fused_sra.h"

#include <cstring>
#include <stdexcept>
#include <string>

#include "../common/a2a.h"
#include "../common/config.h"
#include "../engine/engine.h"  // split_for_fusion
#include "../kernels/launch.h"

namespace cgx {

FusedSra::FusedSra(SymmetricHeap* heap, int max_lanes, int64_t timeout_ms, uint32_t min_lane_elems)
    : heap_(heap), max_lanes_(max_lanes), timeout_ns_((uint64_t)timeout_ms * 1000000ull),
      min_lane_elems_(min_lane_elems) {
  // NVLS: multimem.st for phase B / one-shot, multimem.ld_reduce for raw items (CGX_NVLS=0 disables
  // the heap's multicast mapping altogether; CGX_NVLS_REDUCE=0 keeps the two-shot raw path)
  use_mc_ = heap_->has_multicast() && heap_->world() > 1;
  use_mc_reduce_ = use_mc_ && env_bool("CGX_NVLS_REDUCE", true);
  stages_ = (int)env_int("CGX_STAGES", 0);  // pipeline depth experiment, see pick_stages()
  if (max_lanes_ < 1) max_lanes_ = 1;
  if ((uint32_t)max_lanes_ > heap_->layout().flag_stride) max_lanes_ = (int)heap_->layout().flag_stride;
}

void FusedSra::enable_trace(bool on) {
  trace_on_ = on;
  if (on && d_trace_ == nullptr)
    cuda_check(cudaMalloc((void**)&d_trace_, (size_t)heap_->layout().flag_stride * 8 * sizeof(unsigned long long)),
               "cudaMalloc(trace)");
}

std::vector<uint64_t> FusedSra::read_trace() {
  std::vector<uint64_t> out;
  if (d_trace_ == nullptr || last_lanes_ == 0) return out;
  cuda_check(cudaDeviceSynchronize(), "trace sync");
  out.resize((size_t)last_lanes_ * 8);
  cuda_check(cudaMemcpy(out.data(), d_trace_, out.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost), "trace copy");
  return out;
}

FusedSra::~FusedSra() {
  if (d_trace_) cudaFree(d_trace_);
}

const DevicePlan* FusedSra::prepare(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                                    cudaStream_t stream, int max_lanes) {
  return prepare_impl(layers, dtype, skip_incomplete, stream, world(), heap_->layout().slot_bytes, max_lanes);
}

const DevicePlan* FusedSra::prepare_oneshot(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                                            cudaStream_t stream, int max_lanes) {
  if (heap_->layout().os_slot_bytes == 0) return nullptr;
  return prepare_impl(layers, dtype, skip_incomplete, stream, 1, heap_->layout().os_slot_bytes, max_lanes);
}

const DevicePlan* FusedSra::prepare_impl(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                                         cudaStream_t stream, int plan_world, uint32_t capacity, int max_lanes) {
  PlanOptions opt;
  opt.world = plan_world;
  opt.lanes = (max_lanes > 0 && max_lanes < max_lanes_) ? max_lanes : max_lanes_;
  opt.dtype = dtype;
  opt.skip_incomplete = skip_incomplete;
  opt.min_lane_elems = min_lane_elems_;
  const DevicePlan& dp = plans_.get(layers, opt, stream);
  if (dp.plan.max_chunk_wire > capacity) return nullptr;
  plans_.upload(dp, stream);
  return &dp;
}

namespace {

// an FP8 allreduce: a known codec, compressed blocks of 8 bits only, round to nearest unless the codec
// rounds stochastically
void check_allreduce_codec(const Plan& plan, WireCodec codec, const RngParams& rng) {
  if (codec == kMaxMin) return;
  if (!is_fp8_codec(codec)) throw std::invalid_argument("cgx allreduce: unknown wire codec");
  if (rng.stochastic && !fp8_sr(codec)) throw std::invalid_argument("cgx allreduce: the FP8 formats round to nearest only");
  for (const BlockDesc& d : plan.blocks)
    if (block_bits(d) != 8 && block_bits(d) < kRawBits)
      throw std::invalid_argument("cgx allreduce: an FP8 format needs layers of bits 8 or 32, got " +
                                  std::to_string(block_bits(d)));
}

// split_for_fusion cuts a layer at multiples of its bucket size. A bucket above kMaxBlockElems is
// quantized as kMaxBlockElems-element buckets counted from the layer start, while skip_incomplete
// counts complete buckets of the requested size: such a layer is cut at multiples of both.
std::vector<std::vector<LayerSpec>> split_shard(const std::vector<LayerSpec>& layers, int elsize, int64_t budget) {
  std::vector<LayerSpec> cut = layers;
  for (LayerSpec& l : cut) {
    if (l.bits >= kRawBits || l.bucket <= kMaxBlockElems) continue;
    uint64_t a = l.bucket, b = kMaxBlockElems;
    while (b) {
      const uint64_t t = a % b;
      a = b;
      b = t;
    }
    const uint64_t lcm = (uint64_t)l.bucket / a * kMaxBlockElems;
    if (lcm > 0xFFFFFFFFull) throw std::invalid_argument("cgx reduce_scatter: quantization bucket size too large");
    l.bucket = (uint32_t)lcm;
  }
  std::vector<std::vector<LayerSpec>> groups = split_for_fusion(cut, elsize, budget);
  size_t k = 0;
  for (auto& g : groups)
    for (LayerSpec& s : g) {
      while (s.elem_off >= layers[k].elem_off + layers[k].numel) ++k;
      s.bucket = layers[k].bucket;
    }
  return groups;
}

}  // namespace

void FusedSra::run(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream,
                   WireCodec codec) {
  check_allreduce_codec(dp.plan, codec, rng);
  launch(dp, data, prescale, rng, stream, false, nullptr, 0, false, codec);
}

uint32_t codes_bucket(ShardedOp op, const std::vector<LayerSpec>& shard_layers, WireCodec codec) {
  if (op != ShardedOp::kAllGather)
    throw std::invalid_argument("cgx reduce_scatter: output_scales is an all_gather output");
  if (!is_fp8_codec(codec))
    throw std::invalid_argument("cgx all_gather: output_scales needs an FP8 format (e4m3, e5m2, e4m3_pow2 or e5m2_pow2)");
  const uint32_t B = shard_layers.empty() ? 1u : shard_layers[0].bucket;
  if (B < 1 || B > kMaxBlockElems)
    throw std::invalid_argument("cgx all_gather: output_scales needs 1 <= bucket_size <= " +
                                std::to_string(kMaxBlockElems) + ", got " + std::to_string(B));
  for (const LayerSpec& l : shard_layers) {
    if (l.bits != 8)
      throw std::invalid_argument("cgx all_gather: output_scales needs every layer at bits 8 (raw layers have no codes)");
    if (l.bucket != B || l.numel % B)
      throw std::invalid_argument("cgx all_gather: output_scales needs one bucket_size that divides every layer, got "
                                  "a layer of " + std::to_string(l.numel) + " elements and bucket " +
                                  std::to_string(l.bucket));
  }
  return B;
}

void check_sharded_buffers(ShardedOp op, const std::vector<LayerSpec>& shard_layers, int dtype, const void* in,
                           const void* out, uint64_t S, int rank, int world, WireCodec codec, const float* out_scales) {
  const bool rs = op == ShardedOp::kReduceScatter;
  const char* name = op_name(op);
  if (codec != kMaxMin && !is_fp8_codec(codec))
    throw std::invalid_argument(std::string("cgx ") + name + ": unknown wire codec");
  if (codec != kMaxMin)
    for (const LayerSpec& l : shard_layers)
      if (l.bits != 8 && l.bits < kRawBits)
        throw std::invalid_argument(std::string("cgx ") + name + ": an FP8 format needs layers of bits 8 or 32, got " +
                                    std::to_string(l.bits));
  const uint64_t bucket = out_scales != nullptr ? codes_bucket(op, shard_layers, codec) : 0;
  const uint64_t table = shard_elems(shard_layers);
  if (table != S)
    throw std::invalid_argument(std::string("cgx ") + name + ": the shard layers tile [0, " + std::to_string(table) +
                                ") but the " + (rs ? "output" : "input") + " has " + std::to_string(S) + " elements");
  if (S == 0) return;
  const uint64_t es = (uint64_t)dtype_size(dtype);
  if (out_scales != nullptr) {
    // codes output: S * es input bytes, W * S code bytes, W * S / B fp32 units; the input cannot be
    // a chunk of the codes (the dtypes differ)
    const uintptr_t a = reinterpret_cast<uintptr_t>(in), b = reinterpret_cast<uintptr_t>(out),
                    s = reinterpret_cast<uintptr_t>(out_scales);
    const uint64_t nin = S * es, ncodes = (uint64_t)world * S, nscales = ncodes / bucket * sizeof(float);
    auto overlap = [](uintptr_t x, uint64_t nx, uintptr_t y, uint64_t ny) { return x < y + ny && y < x + nx; };
    if (overlap(a, nin, b, ncodes)) throw std::invalid_argument("cgx all_gather: the codes overlap the input");
    if (overlap(a, nin, s, nscales)) throw std::invalid_argument("cgx all_gather: output_scales overlaps the input");
    if (overlap(b, ncodes, s, nscales)) throw std::invalid_argument("cgx all_gather: output_scales overlaps the codes");
    return;
  }
  const uintptr_t full = reinterpret_cast<uintptr_t>(rs ? in : out);
  const uintptr_t shard = reinterpret_cast<uintptr_t>(rs ? out : in);
  const bool own_chunk = shard == full + (uint64_t)rank * S * es;
  const bool disjoint = shard + S * es <= full || full + (uint64_t)world * S * es <= shard;
  if (!own_chunk && !disjoint)
    throw std::invalid_argument(std::string("cgx ") + name +
                                (rs ? ": the output overlaps the input" : ": the input overlaps the output") +
                                " other than as its chunk " + std::to_string(rank));
}

std::vector<std::vector<LayerSpec>> reduce_scatter_windows(const std::vector<LayerSpec>& shard_layers,
                                                           const PlanOptions& opt, uint32_t slot_bytes) {
  const uint64_t S = shard_elems(shard_layers);
  if (S == 0) return {};
  if (S * (uint64_t)opt.world >= (1ull << 32))
    throw std::invalid_argument("cgx reduce_scatter: the input exceeds 2^32 elements");
  // the largest raw budget whose every window plan fits a slot, halved until it does, starting from
  // the whole shard or the most a slot can carry at 1 bit per element
  const int elsize = dtype_size(opt.dtype);
  for (int64_t budget = (int64_t)std::min<uint64_t>(S * elsize, (uint64_t)slot_bytes * 8 * elsize);; budget /= 2) {
    if (budget < elsize)
      throw std::runtime_error("cgx reduce_scatter: one quantization bucket does not fit the heap slots");
    std::vector<std::vector<LayerSpec>> wins = split_shard(shard_layers, elsize, budget);
    bool fits = true;
    for (const auto& w : wins) fits = fits && build_plan(replicate(w, opt.world, S), opt).max_chunk_wire <= slot_bytes;
    if (fits) return wins;
  }
}

const std::vector<std::vector<LayerSpec>>& FusedSra::rs_windows(const std::vector<LayerSpec>& shard_layers, int dtype,
                                                                bool skip_incomplete, int max_lanes) {
  PlanOptions opt;
  opt.world = world();
  opt.lanes = (max_lanes > 0 && max_lanes < max_lanes_) ? max_lanes : max_lanes_;
  opt.dtype = dtype;
  opt.skip_incomplete = skip_incomplete;
  opt.min_lane_elems = min_lane_elems_;
  const uint64_t key = plan_key(shard_layers, opt);
  auto hit = rs_windows_.find(key);
  if (hit != rs_windows_.end()) return hit->second;
  std::vector<std::vector<LayerSpec>> wins = reduce_scatter_windows(shard_layers, opt, heap_->layout().slot_bytes);
  if (rs_windows_.size() >= kMaxCachedPlans) rs_windows_.clear();
  return rs_windows_.emplace(key, std::move(wins)).first->second;
}

void FusedSra::prepare_sharded(const std::vector<LayerSpec>& shard_layers, int dtype, bool skip_incomplete,
                               cudaStream_t stream, int max_lanes) {
  const uint64_t S = shard_elems(shard_layers);
  for (const auto& w : rs_windows(shard_layers, dtype, skip_incomplete, max_lanes))
    prepare(replicate(w, world(), S), dtype, skip_incomplete, stream, max_lanes);
}

FusedSra::RsCounts FusedSra::sharded(ShardedOp op, const std::vector<LayerSpec>& shard_layers, int dtype,
                                     bool skip_incomplete, const void* in, void* out, uint64_t S, float prescale,
                                     const RngParams& rng, cudaStream_t stream, int max_lanes,
                                     const WindowHook& before_launch, WireCodec codec, float* out_scales) {
  const bool rs = op == ShardedOp::kReduceScatter;
  const char* name = op_name(op);
  RsCounts n;
  check_sharded_buffers(op, shard_layers, dtype, in, out, S, rank(), world(), codec, out_scales);
  const uint32_t out_bucket = out_scales != nullptr ? codes_bucket(op, shard_layers, codec) : 0;
  if (codec != kMaxMin && !fp8_sr(codec) && rng.stochastic)
    throw std::invalid_argument(std::string("cgx ") + name + ": the FP8 formats round to nearest only");
  if (S == 0) return n;
  // plans are launched as soon as they are prepared: a plan-cache trim frees the plans before it
  for (const auto& w : rs_windows(shard_layers, dtype, skip_incomplete, max_lanes)) {
    const DevicePlan* dp = prepare(replicate(w, world(), S), dtype, skip_incomplete, stream, max_lanes);
    if (dp == nullptr)
      throw std::runtime_error(std::string("cgx ") + name + ": window plan does not fit the heap slots");
    if (before_launch) before_launch(w, *dp);
    launch(*dp, const_cast<void*>(in), prescale, rng, stream, false, out, (uint64_t)rank() * S, !rs, codec, out_scales,
           out_bucket);
    const Plan& pl = dp->plan;
    const uint64_t mine = pl.chunk_wire_bytes[rank()], my_elems = pl.chunk_elems[rank()];
    ++n.launches;
    n.elements += pl.numel;
    // the reduce-scatter pushes every chunk but its own, the all-gather its own to W - 1 peers
    n.wire_bytes += rs ? pl.total_wire - mine : mine * (uint64_t)(world() - 1);
    n.raw_bytes += (rs ? pl.numel - my_elems : my_elems * (uint64_t)(world() - 1)) * (uint64_t)dtype_size(dtype);
  }
  return n;
}

void FusedSra::run_oneshot(const DevicePlan& dp, void* data, float prescale, const RngParams& rng,
                           cudaStream_t stream, WireCodec codec) {
  check_allreduce_codec(dp.plan, codec, rng);
  launch(dp, data, prescale, rng, stream, true, nullptr, 0, false, codec);
}

// Pipeline depth of the fused kernel: every chunk's item list can be cut into S pieces, each with
// its own flag value, so that the NVLink flight of one piece overlaps the computation of the next.
// Every extra stage costs one more fence.acq_rel.sys per phase, and a system fence issued while the
// SM keeps streaming peer stores only completes when that traffic drains, so more stages have been
// slower so far. The default therefore stays 1; CGX_STAGES=2..4 keeps the experiment reproducible.
int FusedSra::pick_stages(const DevicePlan&) const {
  const int w = world();
  const int cap = w > 0 ? (32 / w < 4 ? 32 / w : 4) : 1;
  int s = stages_ <= 0 ? 1 : stages_;
  if (s > cap) s = cap;
  return s < 1 ? 1 : s;
}

void FusedSra::launch(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream,
                      bool oneshot, void* out, uint64_t out_shift, bool gather, WireCodec codec, float* out_scales,
                      uint32_t out_bucket) {
  if (!heap_->connected()) throw std::runtime_error("cgx: symmetric heap is not connected");
  if (dp.plan.items.empty()) return;
  ++epoch_;
  SraParams p;
  std::memset(&p, 0, sizeof(p));
  p.data = data;
  p.items = dp.d_items;
  p.item_first = dp.d_item_first;
  p.rank = rank();
  p.world = world();
  p.lanes = dp.plan.lanes;
  p.dtype = dp.plan.dtype;
  p.epoch_hint = epoch_;
  p.prescale = prescale;
  p.rng = make_rng_key(rng, rank(), 0);
  p.slot_bytes = oneshot ? heap_->layout().os_slot_bytes : heap_->layout().slot_bytes;
  p.flag_stride = heap_->layout().flag_stride;
  p.os_parity_stride = (uint32_t)(heap_->layout().os_off[1] - heap_->layout().os_off[0]);
  for (int q = 0; q < kMaxPeers; ++q) {
    const bool valid = q < world();
    // one-shot: recv1 is region 0 of the alternating pair; the kernel adds the parity offset
    p.recv1[q] = valid ? (oneshot ? heap_->oneshot(q, 0) : heap_->recv1(q)) : nullptr;
    p.recv2[q] = valid ? heap_->recv2(q) : nullptr;
    p.flags1[q] = valid ? heap_->flags1(q) : nullptr;
    p.flags2[q] = valid ? heap_->flags2(q) : nullptr;
  }
  // the reduce-scatter kernel uses recv1 and unicast stores only; the all-gather publishes into
  // recv1, through its multicast alias when it has one
  const bool mc = use_mc_ && dp.multicast_ok && (out == nullptr || gather);
  const bool ar = out == nullptr;
  p.mc_recv1 = (mc && oneshot) ? heap_->mc_oneshot(0) : (mc && gather) ? heap_->mc_recv1() : nullptr;
  p.mc_recv2 = (mc && ar && !oneshot) ? heap_->mc_recv2() : nullptr;
  p.mc_reduce = (mc && ar && !oneshot && use_mc_reduce_) ? 1 : 0;
  p.status = heap_->status_device();
  p.abort_word = heap_->abort_device();
  p.timeout_ns = timeout_ns_;
  p.sync = heap_->sync_device();
  p.trace = nullptr;
  if (trace_on_ && d_trace_) {
    // slot 0 takes a minimum, the rest maxima: 0xFF.. / 0 initialisation per lane
    std::vector<unsigned long long> init((size_t)dp.plan.lanes * 8, 0ull);
    for (int l = 0; l < dp.plan.lanes; ++l) init[(size_t)l * 8] = ~0ull;
    cuda_check(cudaMemcpyAsync(d_trace_, init.data(), init.size() * sizeof(unsigned long long),
                               cudaMemcpyHostToDevice, stream),
               "trace init");
    p.trace = d_trace_;
  }
  last_lanes_ = dp.plan.lanes;
  p.uniform_bits = dp.plan.uniform_bits;
  p.slice_elems = (int)dp.plan.slice_elems;
  p.oneshot = oneshot ? 1 : 0;
  p.stages = (oneshot || out != nullptr) ? 1 : pick_stages(dp);
  p.out = out;
  p.out_shift = out_shift;
  p.gather = gather ? 1 : 0;
  // a window of raw layers only has no compressed item: the max-min kernel moves it the same way
  p.codec = dp.plan.uniform_bits == 0 ? kMaxMin : codec;
  p.out_scales = out_scales;
  p.out_bucket = out_bucket;
  cuda_check(launch_sra_fused(p, stream), "launch_sra_fused");
  ++launches_;
}

void check_all_to_all(const void* in, const void* out, const std::vector<uint64_t>& in_counts,
                      const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec, uint32_t bucket,
                      int rank, int world, const A2aRoute* route, const float* out_scales) {
  if ((int)in_counts.size() != world || (int)out_counts.size() != world)
    throw std::invalid_argument("cgx all_to_all: need one input and one output count per rank");
  if (bits < 1 || (bits > 8 && bits < kRawBits))
    throw std::invalid_argument("cgx all_to_all: bits must be in 1..8, or 32 for none");
  if (codec != kMaxMin && !is_fp8_codec(codec))
    throw std::invalid_argument("cgx all_to_all: unknown wire codec");
  if (codec != kMaxMin && bits != 8) throw std::invalid_argument("cgx all_to_all: the FP8 codecs use bits 8");
  if (bucket < 1) throw std::invalid_argument("cgx all_to_all: bucket_size must be >= 1");
  if (in_counts[rank] != out_counts[rank])
    throw std::invalid_argument("cgx all_to_all: a rank's chunk for itself must be as large as the one it receives from itself");
  uint64_t nin = 0, nout = 0;
  for (int q = 0; q < world; ++q) {
    nin += in_counts[q];
    nout += out_counts[q];
  }
  if (nin >= (1ull << 32) || nout >= (1ull << 32))
    throw std::invalid_argument("cgx all_to_all: tensors must have fewer than 2^32 elements");
  if (route != nullptr) {
    const uint64_t row = route->row;
    if (row < 1 || row >= (1ull << 32)) throw std::invalid_argument("cgx all_to_all: rows must have 1 to 2^32 - 1 elements");
    for (int q = 0; q < world; ++q)
      if (in_counts[q] % row || out_counts[q] % row)
        throw std::invalid_argument("cgx all_to_all: with an index, every chunk must be whole rows");
    // the tensors the kernel touches: the indexed ones in full
    if (route->in_index) nin = route->in_rows * row;
    if (route->out_index) nout = route->out_rows * row;
  }
  const uint64_t es = (uint64_t)dtype_size(dtype);
  const uintptr_t a = reinterpret_cast<uintptr_t>(in), b = reinterpret_cast<uintptr_t>(out);
  auto overlap = [](uintptr_t x, uint64_t nx, uintptr_t y, uint64_t ny) { return nx > 0 && ny > 0 && x < y + ny && y < x + nx; };
  if (route != nullptr && route->combine_out != nullptr) {
    const uint64_t k = route->topk;
    if (k < 1 || k > 32) throw std::invalid_argument("cgx all_to_all_combine: top-k must be 1..32");
    if (route->out_index == nullptr) throw std::invalid_argument("cgx all_to_all_combine: needs an output_index");
    if (out_scales != nullptr) throw std::invalid_argument("cgx all_to_all_combine: a codes output (output_scales) has no combine");
    uint64_t entries = 0;
    for (int q = 0; q < world; ++q) entries += out_counts[q] / route->row;
    if (route->out_rows % k || entries != route->out_rows)
      throw std::invalid_argument("cgx all_to_all_combine: output_index must have one entry per slot, T * k = " +
                                  std::to_string(route->out_rows) + " with k = " + std::to_string(k) + ", got " +
                                  std::to_string(entries));
    const uintptr_t c = reinterpret_cast<uintptr_t>(route->combine_out), g = reinterpret_cast<uintptr_t>(route->gate);
    const uint64_t nc = route->out_rows / k * route->row * es, ng = route->out_rows * sizeof(float);
    if (overlap(a, nin * es, c, nc)) throw std::invalid_argument("cgx all_to_all_combine: the output overlaps the input");
    if (overlap(a, nin * es, g, ng)) throw std::invalid_argument("cgx all_to_all_combine: the gate overlaps the input");
    if (overlap(b, nout * es, c, nc)) throw std::invalid_argument("cgx all_to_all_combine: the output overlaps the slots");
  }
  if (route != nullptr && route->in_scale != nullptr) {
    if (route->in_index == nullptr) throw std::invalid_argument("cgx all_to_all: input_scale needs an input_index");
    if (out_scales != nullptr)
      throw std::invalid_argument("cgx all_to_all: input_scale has no codes output (output_scales)");
    if (route->combine_out != nullptr) throw std::invalid_argument("cgx all_to_all: input_scale has no combine (gate)");
    uint64_t sent = 0;
    for (int q = 0; q < world; ++q) sent += in_counts[q] / route->row;
    if (overlap(b, nout * es, reinterpret_cast<uintptr_t>(route->in_scale), sent * sizeof(float)))
      throw std::invalid_argument("cgx all_to_all: input_scale overlaps the output");
  }
  if (out_scales == nullptr) {
    if (overlap(a, nin * es, b, nout * es)) throw std::invalid_argument("cgx all_to_all: the output overlaps the input");
    return;
  }
  // codes output: one byte per output element, one fp32 unit per bucket
  if (codec == kMaxMin) throw std::invalid_argument("cgx all_to_all: output_scales needs an FP8 format (e4m3 or e5m2)");
  if (bucket > kMaxBlockElems)
    throw std::invalid_argument("cgx all_to_all: output_scales needs bucket_size <= " + std::to_string(kMaxBlockElems));
  for (int q = 0; q < world; ++q)
    if (in_counts[q] % bucket || out_counts[q] % bucket)
      throw std::invalid_argument("cgx all_to_all: with output_scales, every chunk must hold whole buckets");
  if (route != nullptr && route->row % bucket)
    throw std::invalid_argument("cgx all_to_all: with output_scales, the row length must be a multiple of bucket_size");
  const uintptr_t s = reinterpret_cast<uintptr_t>(out_scales);
  const uint64_t ns = nout / bucket * sizeof(float);
  if (overlap(a, nin * es, b, nout)) throw std::invalid_argument("cgx all_to_all: the codes overlap the input");
  if (overlap(a, nin * es, s, ns)) throw std::invalid_argument("cgx all_to_all: output_scales overlaps the input");
  if (overlap(b, nout, s, ns)) throw std::invalid_argument("cgx all_to_all: output_scales overlaps the codes");
}

FusedSra::A2aCounts FusedSra::all_to_all(const void* in, void* out, const std::vector<uint64_t>& in_counts,
                                         const std::vector<uint64_t>& out_counts, int dtype, int bits,
                                         WireCodec codec, uint32_t bucket, const RngParams& rng,
                                         cudaStream_t stream, const A2aRoute* route, float* out_scales,
                                         int rank_base) {
  if (!heap_->connected()) throw std::runtime_error("cgx: symmetric heap is not connected");
  const int W = world(), r = rank();
  check_all_to_all(in, out, in_counts, out_counts, dtype, bits, codec, bucket, r, W, route, out_scales);
  if (codec != kMaxMin && !fp8_sr(codec) && rng.stochastic)
    throw std::invalid_argument("cgx all_to_all: the FP8 codecs round to nearest only");
  const uint64_t es = (uint64_t)dtype_size(dtype);
  const bool routed = route != nullptr && (route->in_index != nullptr || route->out_index != nullptr);
  if (routed && route->combine_out != nullptr && route->masks == nullptr)
    throw std::invalid_argument("cgx all_to_all_combine: the fused combine needs its arrival masks");
  if (routed && !a2a_rows_fit((uint32_t)route->row, bits, bucket, (int)es))
    throw std::invalid_argument("cgx all_to_all: rows of " + std::to_string(route->row) +
                                " elements do not hold whole quantization items at this bucket size");
  const int G = max_lanes_;
  const uint32_t lane_slot = a2a_lane_slot_bytes(heap_->layout().slot_bytes, G);
  if (a2a_window_blocks(a2a_geom(0, bits, bucket, (int)es), lane_slot) == 0)
    throw std::invalid_argument("cgx all_to_all: one quantization block does not fit a lane's share of the heap slots "
                                "(raise CGX_FUSION_BUFFER_SIZE_MB)");

  A2aParams p;
  std::memset(&p, 0, sizeof(p));
  p.in = in;
  p.out = out;
  A2aCounts n;
  uint64_t io = 0, oo = 0;
  for (int q = 0; q < W; ++q) {
    p.in_off[q] = (uint32_t)io;
    p.in_cnt[q] = (uint32_t)in_counts[q];
    p.out_off[q] = (uint32_t)oo;
    p.out_cnt[q] = (uint32_t)out_counts[q];
    io += in_counts[q];
    oo += out_counts[q];
    if (q == r || in_counts[q] == 0) continue;
    n.wire_bytes += a2a_chunk_wire(a2a_geom((uint32_t)in_counts[q], bits, bucket, (int)es));
    n.raw_bytes += in_counts[q] * es;
  }
  ++epoch_;
  p.rank = r;
  p.world = W;
  p.lanes = G;
  p.dtype = dtype;
  p.bits = bits >= kRawBits ? kRawBits : bits;
  p.bucket = bucket;
  p.codec = codec;
  p.out_scales = out_scales;
  p.epoch_hint = epoch_;
  p.rng = make_rng_key(rng, r, 0);
  p.rank_base = rank_base;
  p.slot_bytes = heap_->layout().slot_bytes;
  p.lane_slot = lane_slot;
  p.flag_stride = heap_->layout().flag_stride;
  for (int q = 0; q < W; ++q) {
    p.recv[q] = heap_->recv1(q);
    p.flags2[q] = heap_->flags2(q);
    p.landed[q] = heap_->a2a_landed(q);
    p.released[q] = heap_->a2a_released(q);
  }
  p.status = heap_->status_device();
  p.abort_word = heap_->abort_device();
  p.timeout_ns = timeout_ns_;
  p.sync = heap_->sync_device();
  if (routed) {
    p.in_index = route->in_index;
    p.out_index = route->out_index;
    p.row = (uint32_t)route->row;
    p.in_rows = route->in_rows;
    p.out_rows = route->out_rows;
    if (route->combine_out != nullptr) {
      p.combine_out = route->combine_out;
      p.gate = route->gate;
      p.masks = route->masks;
      p.topk = route->topk;
      p.span = a2a_row_span(bits, bucket, (int)es);
    }
    p.in_scale = route->in_scale;
  }
  last_lanes_ = G;
  cudaError_t e = cudaErrorInvalidValue;
  switch (dtype) {
    case kF32: e = launch_a2a_f32(p, stream); break;
    case kF16: e = launch_a2a_f16(p, stream); break;
    case kBF16: e = launch_a2a_bf16(p, stream); break;
    default: break;
  }
  cuda_check(e, "launch_a2a");
  ++launches_;
  n.launches = 1;
  return n;
}

std::string FusedSra::status_message() const {
  const uint32_t s = heap_->status_host();
  if (s == 0) return std::string();
  const uint32_t code = s & 0xFF, peer = (s >> 8) & 0xFF, lane = s >> 16;
  if (code == kSraBadIndex && lane == 2)
    return "cgx: all_to_all on rank " + std::to_string(peer) +
           ": output_index repeats a slot (the combine of its token was skipped; the group refuses further "
           "collectives)";
  if (code == kSraBadIndex)
    return "cgx: all_to_all on rank " + std::to_string(peer) + ": " + (lane ? "output_index" : "input_index") +
           " holds a row outside the " + (lane ? "output" : "input") +
           " (that row was skipped; the group refuses further collectives)";
  if (code == kSraAborted)
    return "cgx: fused allreduce kernel on rank " + std::to_string(rank()) + " was aborted while waiting for rank " +
           std::to_string(peer) + " (lane " + std::to_string(lane) + ")";
  return "cgx: fused allreduce kernel timed out on rank " + std::to_string(rank()) + " waiting for rank " +
         std::to_string(peer) + " (phase " + std::to_string(code) + ", lane " + std::to_string(lane) +
         "); a peer died, is stuck, or issued collectives in a different order "
         "(raise CGX_TIMEOUT_MS if the job is just slow)";
}

void FusedSra::check_status() {
  // sticky: a heap whose kernel gave up is out of step with its peers (epochs, flags) and must
  // not be reused; clear_status() exists for tests that inject faults on purpose
  const std::string msg = status_message();
  if (!msg.empty()) throw std::runtime_error(msg);
}

void FusedSra::clear_status() {
  heap_->clear_status();
  heap_->request_abort(false);
}

}  // namespace cgx

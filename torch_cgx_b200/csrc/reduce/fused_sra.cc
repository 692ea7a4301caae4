#include "fused_sra.h"

#include <cstring>
#include <stdexcept>
#include <string>

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
  for (auto& kv : cache_) {
    if (kv.second->d_items) cudaFree(kv.second->d_items);
    if (kv.second->d_item_first) cudaFree(kv.second->d_item_first);
  }
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
  const uint64_t key = plan_key(layers, opt);
  auto it = cache_.find(key);
  if (it == cache_.end()) {
    if (cache_.size() >= kMaxCachedPlans) {
      // workloads with ever-changing message sizes: drop everything (kernels that still read the
      // old tables are ordered before the frees by the synchronize) and invalidate derived caches
      cuda_check(cudaStreamSynchronize(stream), "sync before trimming the plan cache");
      for (auto& kv : cache_) {
        if (kv.second->d_items) cudaFree(kv.second->d_items);
        if (kv.second->d_item_first) cudaFree(kv.second->d_item_first);
      }
      cache_.clear();
      ++generation_;
    }
    auto dp = std::make_unique<DevicePlan>();
    dp->plan = build_plan(layers, opt);
    {
      bool ok = true;
      for (const BlockDesc& bd : dp->plan.blocks) {
        const int bb = block_bits(bd);
        ok = ok && (block_is_raw(bd) || bb == 2 || bb == 4 || bb == 8);
      }
      dp->multicast_ok = ok;
    }
    if (dp->plan.max_chunk_wire <= capacity && !dp->plan.items.empty()) {
      const size_t ib = dp->plan.items.size() * sizeof(WarpItem);
      const size_t fb = dp->plan.item_first.size() * sizeof(uint32_t);
      cuda_check(cudaMalloc((void**)&dp->d_items, ib), "cudaMalloc(plan items)");
      cuda_check(cudaMalloc((void**)&dp->d_item_first, fb), "cudaMalloc(plan lanes)");
      // pageable source: the runtime stages it before returning, so the vectors may be reused
      cuda_check(cudaMemcpyAsync(dp->d_items, dp->plan.items.data(), ib, cudaMemcpyHostToDevice, stream),
                 "upload plan items");
      cuda_check(cudaMemcpyAsync(dp->d_item_first, dp->plan.item_first.data(), fb, cudaMemcpyHostToDevice, stream),
                 "upload plan lanes");
    }
    if (log_level() >= 2) log_msg(2, "cgx[%d]: new plan %s", rank(), describe_plan(dp->plan).c_str());
    it = cache_.emplace(key, std::move(dp)).first;
  }
  const DevicePlan* dp = it->second.get();
  if (dp->plan.max_chunk_wire > capacity) return nullptr;
  return dp;
}

void FusedSra::run(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream) {
  launch(dp, data, prescale, rng, stream, false);
}

namespace {

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
                                     const RngParams& rng, cudaStream_t stream, int max_lanes) {
  const bool rs = op == ShardedOp::kReduceScatter;
  const char* name = op_name(op);
  RsCounts n;
  const uint64_t table = shard_elems(shard_layers);
  if (table != S)
    throw std::invalid_argument(std::string("cgx ") + name + ": the shard layers tile [0, " + std::to_string(table) +
                                ") but the " + (rs ? "output" : "input") + " has " + std::to_string(S) + " elements");
  if (S == 0) return n;
  {
    const uint64_t es = (uint64_t)dtype_size(dtype);
    const uintptr_t full = reinterpret_cast<uintptr_t>(rs ? in : out);
    const uintptr_t shard = reinterpret_cast<uintptr_t>(rs ? out : in);
    const bool own_chunk = shard == full + (uint64_t)rank() * S * es;
    const bool disjoint = shard + S * es <= full || full + (uint64_t)world() * S * es <= shard;
    if (!own_chunk && !disjoint)
      throw std::invalid_argument(std::string("cgx ") + name +
                                  (rs ? ": the output overlaps the input" : ": the input overlaps the output") +
                                  " other than as its chunk " + std::to_string(rank()));
  }
  // plans are launched as soon as they are prepared: a plan-cache trim frees the plans before it
  for (const auto& w : rs_windows(shard_layers, dtype, skip_incomplete, max_lanes)) {
    const DevicePlan* dp = prepare(replicate(w, world(), S), dtype, skip_incomplete, stream, max_lanes);
    if (dp == nullptr)
      throw std::runtime_error(std::string("cgx ") + name + ": window plan does not fit the heap slots");
    launch(*dp, const_cast<void*>(in), prescale, rng, stream, false, out, (uint64_t)rank() * S, !rs);
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
                           cudaStream_t stream) {
  launch(dp, data, prescale, rng, stream, true);
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
                      bool oneshot, void* out, uint64_t out_shift, bool gather) {
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
  cuda_check(launch_sra_fused(p, stream), "launch_sra_fused");
  ++launches_;
}

std::string FusedSra::status_message() const {
  const uint32_t s = heap_->status_host();
  if (s == 0) return std::string();
  const uint32_t code = s & 0xFF, peer = (s >> 8) & 0xFF, lane = s >> 16;
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

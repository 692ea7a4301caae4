#include "engine.h"

#include "../common/nvtx.h"

#include <algorithm>
#include <stdexcept>

namespace cgx {

std::vector<std::vector<LayerSpec>> split_for_fusion(const std::vector<LayerSpec>& layers, int elsize,
                                                     int64_t fusion_bytes) {
  std::vector<std::vector<LayerSpec>> groups;
  const uint64_t cap = std::max<uint64_t>(1, (uint64_t)fusion_bytes / (uint64_t)elsize);
  std::vector<LayerSpec> cur;
  uint64_t cur_elems = 0;
  auto flush = [&]() {
    if (!cur.empty()) groups.push_back(std::move(cur));
    cur.clear();
    cur_elems = 0;
  };
  for (const LayerSpec& l : layers) {
    if (l.numel == 0) continue;
    if (l.numel > cap) {
      // slice a huge layer at bucket-aligned boundaries, each slice its own call
      flush();
      const uint64_t gran = (l.bits >= kRawBits) ? 512 : std::max<uint32_t>(1u, l.bucket);
      uint64_t step = std::max<uint64_t>(gran, cap / gran * gran);
      for (uint64_t off = 0; off < l.numel; off += step) {
        LayerSpec s = l;
        s.elem_off = l.elem_off + off;
        s.numel = std::min<uint64_t>(step, l.numel - off);
        groups.push_back({s});
      }
      continue;
    }
    if (cur_elems + l.numel > cap) flush();
    cur.push_back(l);
    cur_elems += l.numel;
  }
  flush();
  return groups;
}

AllreduceEngine::AllreduceEngine(int rank, int world, const EngineConfig& cfg)
    : rank_(rank), world_(world), local_size_(world), cfg_(cfg) {}

AllreduceEngine::~AllreduceEngine() {
  // reducers release their scratch through the block backend: they must go first
  for (GenericPath* g : {&gen_cuda_, &gen_cpu_}) {
    g->cross.reset();
    g->intra.reset();
    g->cross_comm.reset();
    g->intra_comm.reset();
    g->ops.reset();
  }
  fused_.reset();
  heap_.reset();
}

void AllreduceEngine::set_topology(int local_size) {
  if (local_size < 1 || local_size > world_ || world_ % local_size != 0) local_size = world_;
  local_size_ = local_size;
}

void AllreduceEngine::attach_generic(bool cuda, std::unique_ptr<Communicator> intra,
                                     std::unique_ptr<Communicator> cross) {
  GenericPath& g = cuda ? gen_cuda_ : gen_cpu_;
  g.intra.reset();
  g.cross.reset();
  g.ops = cuda ? make_cuda_block_backend() : make_cpu_block_backend();
  g.intra_comm = std::move(intra);
  g.cross_comm = std::move(cross);
  if (g.intra_comm) g.intra = make_reducer(cfg_.inner_reduction, g.intra_comm.get(), g.ops.get());
  if (g.cross_comm) g.cross = make_reducer(cfg_.cross_reduction, g.cross_comm.get(), g.ops.get());
}

size_t AllreduceEngine::required_oneshot_slot_bytes(const EngineConfig& cfg) {
  if (cfg.oneshot_max_bytes <= 0) return 0;
  // whole-buffer image: raw worst case + per-block padding + one block of slack
  return (size_t)cfg.oneshot_max_bytes + (size_t)cfg.oneshot_max_bytes / 8 + (size_t)kMaxBlockElems * 4 + 4096;
}

size_t AllreduceEngine::required_slot_bytes(const EngineConfig& cfg, int world) {
  // a raw chunk of a full fusion buffer + slack for chunk imbalance (one block)
  // and per-block 16 B padding
  size_t per = (size_t)cfg.fusion_bytes / (size_t)world;
  return per + per / 8 + (size_t)kMaxBlockElems * 4 + 4096;
}

void AllreduceEngine::attach_heap(std::unique_ptr<SymmetricHeap> heap, int lanes) {
  heap_ = std::move(heap);
  fused_ = std::make_unique<FusedSra>(heap_.get(), lanes, cfg_.timeout_ms, cfg_.min_lane_elems);
}

void AllreduceEngine::check_health() {
  if (fused_) fused_->check_status();
}

static std::vector<LayerSpec> resolve_layers(int64_t numel, const EngineConfig& cfg, const CompressionEnv& env,
                                             int explicit_bucket) {
  int64_t n_eff = numel;
  if (cfg.fake_ratio < 1.0) n_eff = std::max<int64_t>(1, (int64_t)((double)numel * cfg.fake_ratio));
  int resolved = -1;
  return LayerRegistry::instance().extract(n_eff, env, cfg.min_compress_elems, explicit_bucket, &resolved);
}

void AllreduceEngine::launch_fused(const Launch& l, void* data, float prescale, RngParams rng, cudaStream_t stream) {
  const int elsize = dtype_size(l.dp->plan.dtype);
  rng.seq = (rng.seq << 3) | (l.rng_sub & 7u);
  const int lw = fused_->world(), lr = fused_->rank();
  if (l.oneshot) {
    fused_->run_oneshot(*l.dp, data, prescale, rng, stream);
    stats_.wire_bytes += l.dp->plan.total_wire * (uint64_t)(lw - 1);
    stats_.raw_bytes += l.dp->plan.numel * (uint64_t)elsize * (uint64_t)(lw - 1);
  } else {
    fused_->run(*l.dp, data, prescale, rng, stream);
    // bytes pushed by this rank: phase A = every chunk but mine, phase B = mine to W-1 peers
    const uint64_t mine = l.dp->plan.chunk_wire_bytes[lr];
    stats_.wire_bytes += (l.dp->plan.total_wire - mine) + mine * (uint64_t)(lw - 1);
    const uint64_t my_elems = l.dp->plan.chunk_elems[lr];
    stats_.raw_bytes += ((l.dp->plan.numel - my_elems) + my_elems * (uint64_t)(lw - 1)) * (uint64_t)elsize;
  }
  ++stats_.kernel_launches;
  stats_.elements += l.dp->plan.numel;
  if (recording_) recording_->push_back(l);
}

void AllreduceEngine::allreduce_cuda(void* data, int dtype, int64_t numel, bool average, int explicit_bucket,
                                     cudaStream_t stream, bool overlapped) {
  if (numel <= 0) return;
  NvtxRange range("cgx:allreduce_cuda", (uint64_t)numel);
  CompressionEnv env = CompressionEnv::read();
  const bool cacheable = explicit_bucket >= 0 && explicit_bucket < 4096 && nodes() == 1 && fused_ &&
                         cfg_.inner_comm == CommType::kP2P && !cfg_.dummy_compression && cfg_.fake_ratio >= 1.0;
  if (cacheable) {
    if ((size_t)explicit_bucket >= fast_.size()) fast_.resize((size_t)explicit_bucket + 1);
    BucketFast& f = fast_[(size_t)explicit_bucket];
    const uint64_t ver = LayerRegistry::instance().version();
    if (f.registry_version == ver && f.plan_generation == fused_->generation() && f.numel == numel &&
        f.dtype == dtype && f.env_bits == env.bits && f.env_bucket == env.bucket_size &&
        f.skip_incomplete == env.skip_incomplete && f.overlapped == overlapped && !f.launches.empty()) {
      fused_->check_status();
      ++call_seq_;
      ++stats_.calls;
      RngParams rng;
      rng.seed = env.seed;
      rng.stochastic = env.stochastic;
      const float prescale = average ? 1.0f / (float)world_ : 1.0f;
      uint32_t sub = 0;
      const DevicePlan* prev_group = nullptr;
      (void)prev_group;
      for (const Launch& l : f.launches) {
        rng.seq = (call_seq_ << 4) | ((sub++) & 15u);
        launch_fused(l, data, prescale, rng, stream);
      }
      return;
    }
    // slow path once, recording what was launched. A plan-cache trim in the middle of the call
    // (generation bump) frees the plans recorded so far: keep the recording only if none happened.
    std::vector<Launch> rec;
    recording_ = &rec;
    const uint64_t gen_before = fused_->generation();
    try {
      allreduce_cuda_layers(data, dtype, resolve_layers(numel, cfg_, env, explicit_bucket), average, env, stream,
                            overlapped);
    } catch (...) {
      recording_ = nullptr;
      throw;
    }
    recording_ = nullptr;
    if (fused_->generation() != gen_before) {
      f.launches.clear();
      return;
    }
    f.registry_version = ver;
    f.plan_generation = fused_->generation();
    f.numel = numel;
    f.dtype = dtype;
    f.env_bits = env.bits;
    f.env_bucket = env.bucket_size;
    f.skip_incomplete = env.skip_incomplete;
    f.overlapped = overlapped;
    f.launches = std::move(rec);
    return;
  }
  allreduce_cuda_layers(data, dtype, resolve_layers(numel, cfg_, env, explicit_bucket), average, env, stream,
                        overlapped);
}

void AllreduceEngine::sharded_cuda(ShardedOp op, const void* in, void* out, int dtype, int64_t shard_numel,
                                   std::vector<LayerSpec> shard_layers, bool average, int bits, int bucket,
                                   bool skip_incomplete, const RngParams& rng_in, cudaStream_t stream,
                                   bool overlapped) {
  if (nodes() > 1)
    throw std::runtime_error(std::string("cgx: the compressed ") + op_title(op) + " supports a single node only");
  if (!fused_ || cfg_.inner_comm != CommType::kP2P)
    throw std::runtime_error(std::string("cgx: the compressed ") + op_title(op) +
                             " needs the P2P transport (CGX_INNER_COMMUNICATOR_TYPE=P2P)");
  fused_->check_status();
  if (shard_numel <= 0) return;
  NvtxRange range(op == ShardedOp::kReduceScatter ? "cgx:reduce_scatter_cuda" : "cgx:all_gather_cuda",
                  (uint64_t)shard_numel);
  if (shard_layers.empty()) {
    LayerSpec l;
    l.elem_off = 0;
    l.numel = (uint64_t)shard_numel;
    l.bits = compression_enabled(shard_numel, bits, cfg_.min_compress_elems) ? bits : kRawBits;
    l.bucket = (uint32_t)std::max(1, bucket);
    shard_layers.push_back(l);
  }
  ++call_seq_;
  ++stats_.calls;
  RngParams rng = rng_in;
  rng.seq = call_seq_ << 4;  // one sequence for every window: the counters are element indices of the full buffer
  const FusedSra::RsCounts n =
      fused_->sharded(op, shard_layers, dtype, skip_incomplete, in, out, (uint64_t)shard_numel,
                      average ? 1.0f / (float)world_ : 1.0f, rng, stream, overlapped ? cfg_.overlap_lanes : 0);
  stats_.kernel_launches += n.launches;
  stats_.elements += n.elements;
  stats_.wire_bytes += n.wire_bytes;
  stats_.raw_bytes += n.raw_bytes;
}

void AllreduceEngine::allreduce_cpu(void* data, int dtype, int64_t numel, bool average, int explicit_bucket) {
  if (numel <= 0) return;
  allreduce_cpu_prepared(data, dtype, prepare_cpu(numel, explicit_bucket), average);
}

AllreduceEngine::CpuCall AllreduceEngine::prepare_cpu(int64_t numel, int explicit_bucket) const {
  CpuCall c;
  c.env = CompressionEnv::read();
  if (numel > 0) c.layers = resolve_layers(numel, cfg_, c.env, explicit_bucket);
  return c;
}

void AllreduceEngine::allreduce_cpu_prepared(void* data, int dtype, const CpuCall& call, bool average) {
  if (call.layers.empty()) return;
  if (!gen_cpu_.ops) throw std::runtime_error("cgx: CPU reducers are not initialised");
  // one host reduction at a time: the worker thread and a caller-thread CUDA call share counters
  std::lock_guard<std::mutex> g(cpu_mu_);
  NvtxRange range("cgx:allreduce_cpu", (uint64_t)call.layers.size());
  run_layers(false, data, dtype, call.layers, average, call.env, nullptr);
}

void AllreduceEngine::allreduce_cuda_layers(void* data, int dtype, const std::vector<LayerSpec>& layers_in,
                                            bool average, const CompressionEnv& env, cudaStream_t stream,
                                            bool overlapped) {
  const bool need_fused = cfg_.inner_comm == CommType::kP2P && local_size_ > 0;
  if (need_fused && !fused_) throw std::runtime_error("cgx: P2P path is not initialised");
  if (fused_) fused_->check_status();
  lane_cap_ = overlapped ? cfg_.overlap_lanes : 0;
  try {
    run_layers(true, data, dtype, layers_in, average, env, stream);
  } catch (...) {
    lane_cap_ = 0;
    throw;
  }
  lane_cap_ = 0;
}

// One node-local allreduce of a fusion group: fused P2P kernel when available,
// otherwise the generic reducer over the intra-node communicator.
void AllreduceEngine::intra_stage(bool cuda, void* data, int dtype, const std::vector<LayerSpec>& group,
                                  bool skip_incomplete, float prescale, RngParams rng, cudaStream_t stream) {
  GenericPath& g = cuda ? gen_cuda_ : gen_cpu_;
  const int elsize = dtype_size(dtype);
  // the fused kernel implements SRA (+ the one-shot variant); an explicitly requested Ring or
  // all-to-all intra-node reduction goes through the generic reducers instead
  const bool want_fused = cfg_.inner_reduction == ReductionType::kSRA || !g.intra;
  if (cuda && fused_ && cfg_.inner_comm == CommType::kP2P && want_fused) {
    // latency-bound messages: single-hop one-shot kernel
    if (fused_->world() > 1 && cfg_.oneshot_max_bytes > 0) {
      uint64_t n = 0;
      for (const LayerSpec& l : group) n += l.numel;
      if ((int64_t)(n * (uint64_t)elsize) <= cfg_.oneshot_max_bytes) {
        const DevicePlan* dp = fused_->prepare_oneshot(group, dtype, skip_incomplete, stream, lane_cap_);
        // every rank pushes its whole packed image to W-1 peers: keep that egress small
        if (dp != nullptr && dp->plan.total_wire * (uint64_t)(fused_->world() - 1) <= (4ull << 20)) {
          launch_fused(Launch{dp, true, 0u}, data, prescale, rng, stream);
          return;
        }
      }
    }
    // work list; a group whose plan does not fit the heap slots is halved
    std::vector<std::vector<LayerSpec>> todo{group};
    uint32_t sub = 0;
    while (!todo.empty()) {
      std::vector<LayerSpec> gl = std::move(todo.back());
      todo.pop_back();
      const DevicePlan* dp = fused_->prepare(gl, dtype, skip_incomplete, stream, lane_cap_);
      if (dp == nullptr) {
        if (gl.size() > 1) {
          size_t half = gl.size() / 2;
          std::vector<LayerSpec> a(gl.begin(), gl.begin() + half), b(gl.begin() + half, gl.end());
          todo.push_back(std::move(b));
          todo.push_back(std::move(a));
        } else {
          const LayerSpec& l = gl[0];
          const uint64_t gran = (l.bits >= kRawBits) ? 512 : std::max<uint32_t>(1u, l.bucket);
          if (l.numel <= gran)
            throw std::runtime_error("cgx: fusion buffer too small for a single quantization bucket");
          uint64_t h = std::max<uint64_t>(gran, (l.numel / 2) / gran * gran);
          LayerSpec a = l, b = l;
          a.numel = h;
          b.elem_off = l.elem_off + h;
          b.numel = l.numel - h;
          todo.push_back({b});
          todo.push_back({a});
        }
        continue;
      }
      launch_fused(Launch{dp, false, sub++}, data, prescale, rng, stream);
    }
    return;
  }
  if (g.intra) {
    const uint64_t before = g.intra->bytes_sent();
    g.intra->allreduce(data, dtype, group, skip_incomplete, prescale, rng, stream);
    stats_.wire_bytes += g.intra->bytes_sent() - before;
    uint64_t n = 0;
    for (const LayerSpec& l : group) n += l.numel;
    stats_.elements += n;
    const int lw = local_size_;
    stats_.raw_bytes += 2ull * n * (uint64_t)elsize * (uint64_t)(lw - 1) / (uint64_t)lw;
    return;
  }
  if (local_size_ > 1) throw std::runtime_error("cgx: no intra-node reducer available for this tensor");
}

void AllreduceEngine::run_layers(bool cuda, void* data, int dtype, std::vector<LayerSpec> layers, bool average,
                                 const CompressionEnv& env, cudaStream_t stream) {
  GenericPath& g = cuda ? gen_cuda_ : gen_cpu_;
  if (cfg_.dummy_compression)
    for (LayerSpec& l : layers) l.bits = kRawBits;
  const int elsize = dtype_size(dtype);
  const float prescale = average ? 1.0f / (float)world_ : 1.0f;
  ++call_seq_;
  ++stats_.calls;
  RngParams rng;
  rng.seed = env.seed;
  rng.stochastic = env.stochastic;
  const bool multi_node = nodes() > 1;
  if (multi_node && !g.cross) throw std::runtime_error("cgx: multi-node topology but no cross-node reducer");

  uint32_t sub = 0;
  for (std::vector<LayerSpec>& group : split_for_fusion(layers, elsize, cfg_.fusion_bytes)) {
    rng.seq = (call_seq_ << 4) | (sub++ & 15u);
    // ---- stage 1: inside the node (reference: mpi_allreduce_operations.cc:146-160)
    std::vector<LayerSpec> intra_layers = group;
    if (!cfg_.intra_compress && multi_node)
      for (LayerSpec& l : intra_layers) l.bits = kRawBits;
    if (local_size_ > 1 || !multi_node) {
      NvtxRange r1("cgx:intra_node", (uint64_t)intra_layers.size());
      intra_stage(cuda, data, dtype, intra_layers, env.skip_incomplete, prescale, rng, stream);
    }
    if (!multi_node) continue;
    NvtxRange r2("cgx:cross_node", (uint64_t)group.size());
    // ---- stage 2: across nodes (reference: mpi_allreduce_operations.cc:161-183)
    RngParams crng = rng;
    crng.seq = rng.seq ^ 0x40000000u;
    const float cross_scale = (local_size_ > 1) ? 1.0f : prescale;
    if (cfg_.intra_broadcast && local_size_ > 1) {
      if (local_rank() == 0) g.cross->allreduce(data, dtype, group, env.skip_incomplete, cross_scale, crng, stream);
      // leaders hand the result to the rest of their node: packed when the intra-node stage
      // compresses (reference: Reducer::Broadcast with do_compression && intra_compress_,
      // mpi_allreduce_operations.cc:171-176, reducer.cc:96-160), raw bytes of the span otherwise
      bool any_compressed = false;
      for (const LayerSpec& l : group) any_compressed = any_compressed || l.bits < kRawBits;
      if (g.intra && cfg_.intra_compress && any_compressed) {
        RngParams brng = rng;
        brng.seq = rng.seq ^ 0x20000000u;
        const uint64_t before = g.intra->bytes_sent();
        g.intra->broadcast_compressed(data, dtype, group, env.skip_incomplete, 0, brng, stream);
        stats_.wire_bytes += g.intra->bytes_sent() - before;
      } else {
        uint64_t lo = ~0ull, hi = 0;
        for (const LayerSpec& l : group) {
          lo = std::min<uint64_t>(lo, l.elem_off);
          hi = std::max<uint64_t>(hi, l.elem_off + l.numel);
        }
        if (hi > lo && g.intra)
          g.intra->broadcast(static_cast<uint8_t*>(data) + lo * elsize, (size_t)(hi - lo) * elsize, 0, stream);
      }
    } else {
      g.cross->allreduce(data, dtype, group, env.skip_incomplete, cross_scale, crng, stream);
    }
  }
}

}  // namespace cgx

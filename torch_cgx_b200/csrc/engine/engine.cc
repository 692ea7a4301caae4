#include "engine.h"

#include "../common/a2a.h"
#include "../common/nvtx.h"

#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <string>

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

namespace {
// the communicator of a one-rank group: there is no one to exchange with
class SelfCommunicator : public Communicator {
 public:
  explicit SelfCommunicator(bool cuda) : cuda_(cuda) {}
  int rank() const override { return 0; }
  int size() const override { return 1; }
  bool is_cuda() const override { return cuda_; }
  void exchange(const std::vector<P2POp>& ops, cudaStream_t) override {
    if (!ops.empty()) throw std::logic_error("cgx: a one-rank group has no peer to exchange with");
  }
  void barrier() override {}

 private:
  bool cuda_;
};
}  // namespace

AllreduceEngine::AllreduceEngine(int rank, int world, const EngineConfig& cfg)
    : rank_(rank), world_(world), local_size_(world), cfg_(cfg) {}

AllreduceEngine::~AllreduceEngine() {
  // reducers release their scratch through the block backend: they must go first
  for (GenericPath* g : {&gen_cuda_, &gen_cpu_}) {
    for (GenericPath::Buf* b : {&g->a2a_send, &g->a2a_recv})
      if (b->p) g->ops->release(b->p);
    g->world_comm.reset();
    g->self.reset();
    g->self_comm.reset();
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
  g.self.reset();
  g.self_comm.reset();
  g.intra.reset();
  g.cross.reset();
  g.ops = cuda ? make_cuda_block_backend() : make_cpu_block_backend();
  g.intra_comm = std::move(intra);
  g.cross_comm = std::move(cross);
  if (g.intra_comm) g.intra = make_reducer(cfg_.inner_reduction, g.intra_comm.get(), g.ops.get());
  if (g.cross_comm) g.cross = make_reducer(cfg_.cross_reduction, g.cross_comm.get(), g.ops.get());
}

void AllreduceEngine::attach_world(bool cuda, std::unique_ptr<Communicator> world) {
  GenericPath& g = cuda ? gen_cuda_ : gen_cpu_;
  if (!g.ops) throw std::logic_error("cgx: attach_world needs attach_generic first");
  if (world && (world->size() != world_ || world->rank() != rank_))
    throw std::invalid_argument("cgx: the world communicator must span the world, with this rank's world rank");
  g.world_comm = std::move(world);
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

void AllreduceEngine::launch_fused(const Launch& l, void* data, float prescale, RngParams rng, cudaStream_t stream,
                                   WireCodec codec, const std::vector<LayerSpec>* layers) {
  const int elsize = dtype_size(l.dp->plan.dtype);
  rng.seq = (rng.seq << 3) | (l.rng_sub & 7u);
  const int lw = fused_->world(), lr = fused_->rank();
  if (observer_) {
    observer_->stage(EngineStage{l.oneshot ? EngineStage::kOneshot : EngineStage::kSra, layers, l.dp, rng, prescale});
    observer_->before_fused_launch(*l.dp, stream);
  }
  if (l.oneshot) {
    fused_->run_oneshot(*l.dp, data, prescale, rng, stream, codec);
    stats_.wire_bytes += l.dp->plan.total_wire * (uint64_t)(lw - 1);
    stats_.raw_bytes += l.dp->plan.numel * (uint64_t)elsize * (uint64_t)(lw - 1);
  } else {
    fused_->run(*l.dp, data, prescale, rng, stream, codec);
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
                                     cudaStream_t stream, bool overlapped, std::optional<WireCodec> codec) {
  if (numel <= 0) return;
  NvtxRange range("cgx:allreduce_cuda", (uint64_t)numel);
  CompressionEnv env = CompressionEnv::read();
  if (codec) env.codec = *codec;
  const bool cacheable = explicit_bucket >= 0 && explicit_bucket < 4096 && nodes() == 1 && fused_ &&
                         cfg_.inner_comm == CommType::kP2P && !cfg_.dummy_compression && cfg_.fake_ratio >= 1.0;
  if (cacheable) {
    if ((size_t)explicit_bucket >= fast_.size()) fast_.resize((size_t)explicit_bucket + 1);
    BucketFast& f = fast_[(size_t)explicit_bucket];
    const uint64_t ver = LayerRegistry::instance().version();
    if (f.registry_version == ver && f.plan_generation == fused_->generation() && f.numel == numel &&
        f.dtype == dtype && f.env_bits == env.bits && f.env_bucket == env.bucket_size && f.env_codec == env.codec &&
        f.skip_incomplete == env.skip_incomplete && f.overlapped == overlapped && !f.launches.empty()) {
      fused_->check_status();
      ++call_seq_;
      ++stats_.calls;
      RngParams rng;
      rng.seed = env.seed;
      rng.stochastic = env.stochastic;
      const float prescale = average ? 1.0f / (float)world_ : 1.0f;
      // the sequence numbers of the slow path: fusion group in the call's, piece in the launch's
      for (const Launch& l : f.launches) {
        rng.seq = (call_seq_ << 4) | (l.rng_group & 15u);
        launch_fused(l, data, prescale, rng, stream, (WireCodec)env.codec);
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
    f.env_codec = env.codec;
    f.skip_incomplete = env.skip_incomplete;
    f.overlapped = overlapped;
    f.launches = std::move(rec);
    return;
  }
  allreduce_cuda_layers(data, dtype, resolve_layers(numel, cfg_, env, explicit_bucket), average, env, stream,
                        overlapped);
}

std::vector<LayerSpec> AllreduceEngine::sharded_table(int64_t shard_numel, std::vector<LayerSpec> layers, int bits,
                                                      int bucket) const {
  if (layers.empty() && shard_numel > 0) {
    LayerSpec l;
    l.elem_off = 0;
    l.numel = (uint64_t)shard_numel;
    l.bits = compression_enabled(shard_numel, bits, cfg_.min_compress_elems) ? bits : kRawBits;
    l.bucket = (uint32_t)std::max(1, bucket);
    layers.push_back(l);
  }
  return layers;
}

std::vector<LayerSpec> AllreduceEngine::sharded_intra_table(ShardedOp op, std::vector<LayerSpec> table) const {
  if (nodes() > 1 && (op == ShardedOp::kAllGather || !cfg_.intra_compress))
    for (LayerSpec& l : table) l.bits = kRawBits;
  return table;
}

void AllreduceEngine::prepare_sharded(ShardedOp op, const std::vector<LayerSpec>& shard_layers, int dtype,
                                      bool skip_incomplete, cudaStream_t stream) {
  if (fused_) fused_->prepare_sharded(sharded_intra_table(op, shard_layers), dtype, skip_incomplete, stream);
}

void AllreduceEngine::sharded_intra(bool cuda, ShardedOp op, const void* in, void* out, int dtype, uint64_t S,
                                    const std::vector<LayerSpec>& table, bool skip_incomplete, float prescale,
                                    const RngParams& rng, cudaStream_t stream, bool overlapped, WireCodec codec,
                                    float* out_scales) {
  const bool rs = op == ShardedOp::kReduceScatter;
  if (fused_sharded(cuda)) {
    FusedSra::WindowHook hook;
    if (observer_)
      hook = [&](const std::vector<LayerSpec>& w, const DevicePlan& dp) {
        observer_->stage(EngineStage{rs ? EngineStage::kRs : EngineStage::kAg, &w, &dp, rng, prescale});
        observer_->before_fused_launch(dp, stream);
      };
    const FusedSra::RsCounts n = fused_->sharded(op, table, dtype, skip_incomplete, in, out, S, prescale, rng,
                                                 stream, overlapped ? cfg_.overlap_lanes : 0, hook, codec,
                                                 out_scales);
    stats_.kernel_launches += n.launches;
    stats_.elements += n.elements;
    stats_.wire_bytes += n.wire_bytes;
    stats_.raw_bytes += n.raw_bytes;
    return;
  }
  GenericPath& g = cuda ? gen_cuda_ : gen_cpu_;
  const uint64_t before = g.intra->bytes_sent();
  observe(rs ? EngineStage::kGenericRs : EngineStage::kGenericAg, &table, rng, prescale);
  if (rs)
    g.intra->reduce_scatter(in, out, dtype, table, skip_incomplete, prescale, rng, stream, codec);
  else
    g.intra->all_gather(in, out, dtype, table, skip_incomplete, rng, stream, codec, out_scales);
  // the fused kernel's conventions: the elements of the window, the raw bytes a raw exchange would move
  const uint64_t L = (uint64_t)local_size_, es = (uint64_t)dtype_size(dtype);
  stats_.wire_bytes += g.intra->bytes_sent() - before;
  stats_.elements += L * S;
  stats_.raw_bytes += S * (L - 1) * es;
}

// Two stages when there are several nodes (DESIGN §2.9b), N = nodes(), L = local_size_, r = n * L + l:
//  reduce-scatter: 1. per node block b, the node-local reduce-scatter of in[b*L*S, (b+1)*L*S) into
//                     staging[b*S, (b+1)*S) (the node's partial of chunk b*L + l), prescaled by 1/W;
//                  2. the cross-node reduce-scatter of the N partials among the ranks of local rank l,
//                     prescale 1 (1/W and straight from `in` when L = 1).
//  all-gather:     1. the cross-node all-gather of the shard into staging (into `out` when L = 1);
//                  2. per node n', the node-local all-gather of staging[n'*S, (n'+1)*S) into
//                     out[n'*L*S, (n'+1)*L*S) with a raw table: every shard is quantized once.
// RNG sequences: node block b runs with call_seq << 4 ^ b (one node: today's call_seq << 4), the
// cross-node stage with call_seq << 4 ^ 0x40000000, the allreduce's cross-node marker.
void AllreduceEngine::sharded(bool cuda, ShardedOp op, const void* in, void* out, void* staging, int dtype,
                              int64_t shard_numel, const std::vector<LayerSpec>& shard_layers, bool average,
                              bool skip_incomplete, const RngParams& rng_in, cudaStream_t stream, bool overlapped,
                              WireCodec codec, float* out_scales) {
  GenericPath& g = cuda ? gen_cuda_ : gen_cpu_;
  const int N = nodes(), L = local_size_;
  const std::string title = std::string("cgx: the compressed ") + op_title(op);
  // every rank evaluates the same condition, so every rank refuses and none is left waiting
  if (out_scales != nullptr && N > 1)
    throw std::runtime_error(title + " with output_scales runs on one node only (CGX_LOCAL_SIZE " +
                             std::to_string(L) + " < world size " + std::to_string(world_) + ")");
  const bool fused = fused_sharded(cuda);
  if (fused) fused_->check_status();
  if (shard_numel <= 0) return;
  check_sharded_buffers(op, shard_layers, dtype, in, out, (uint64_t)shard_numel, rank_, world_, codec, out_scales);
  if (codec != kMaxMin && !fp8_sr(codec) && rng_in.stochastic)
    throw std::invalid_argument(title + ": the FP8 formats round to nearest only");
  if (!fused && (L > 1 || N == 1) && !g.intra)
    throw std::runtime_error(title + (L > 1 ? " has no intra-node reducer" : " of one rank needs the P2P transport"));
  if (N > 1 && !g.cross) throw std::runtime_error(title + ": multi-node topology but no cross-node reducer");
  if (sharded_staging_numel(shard_numel) > 0 && staging == nullptr)
    throw std::runtime_error(title + ": several nodes need a staging buffer");
  NvtxRange range(op == ShardedOp::kReduceScatter ? "cgx:reduce_scatter_cuda" : "cgx:all_gather_cuda",
                  (uint64_t)shard_numel);
  ++call_seq_;
  ++stats_.calls;
  const uint64_t S = (uint64_t)shard_numel;
  const size_t shard_bytes = (size_t)S * (size_t)dtype_size(dtype);
  const float prescale = average ? 1.0f / (float)world_ : 1.0f;
  const uint32_t seq = call_seq_ << 4;  // one sequence for every window: the counters are element indices
  RngParams rng = rng_in, crng = rng_in;
  crng.seq = seq ^ 0x40000000u;
  const std::vector<LayerSpec> intra_table = sharded_intra_table(op, shard_layers);
  const bool intra = L > 1 || N == 1;
  auto at = [](const void* p, size_t off) { return static_cast<uint8_t*>(const_cast<void*>(p)) + off; };
  if (op == ShardedOp::kReduceScatter) {
    void* partial = N > 1 ? staging : out;
    if (intra)
      for (int b = 0; b < N; ++b) {
        rng.seq = seq ^ (uint32_t)b;
        NvtxRange r1("cgx:intra_node", (uint64_t)b);
        sharded_intra(cuda, op, at(in, (size_t)b * L * shard_bytes), at(partial, (size_t)b * shard_bytes), dtype, S,
                      intra_table, skip_incomplete, prescale, rng, stream, overlapped, codec);
      }
    if (N == 1) return;
    NvtxRange r2("cgx:cross_node", (uint64_t)N);
    const float cross_scale = L > 1 ? 1.0f : prescale;
    observe(EngineStage::kCrossRs, &shard_layers, crng, cross_scale);
    g.cross->reduce_scatter(L > 1 ? partial : in, out, dtype, shard_layers, skip_incomplete, cross_scale, crng, stream,
                            codec);
    return;
  }
  void* gathered = L > 1 ? staging : out;
  if (N > 1) {
    NvtxRange r2("cgx:cross_node", (uint64_t)N);
    observe(EngineStage::kCrossAg, &shard_layers, crng, 1.0f);
    g.cross->all_gather(in, gathered, dtype, shard_layers, skip_incomplete, crng, stream, codec);
  }
  if (!intra) return;
  for (int n = 0; n < N; ++n) {
    rng.seq = seq ^ (uint32_t)n;
    NvtxRange r1("cgx:intra_node", (uint64_t)n);
    sharded_intra(cuda, op, N > 1 ? at(gathered, (size_t)n * shard_bytes) : in,
                  at(out, (size_t)n * L * shard_bytes), dtype, S, intra_table, skip_incomplete, 1.0f, rng, stream,
                  overlapped, codec, out_scales);
  }
}

void AllreduceEngine::all_to_all(bool cuda, const void* in, void* out, const std::vector<uint64_t>& in_counts,
                                 const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec,
                                 uint32_t bucket, const RngParams& rng_in, cudaStream_t stream,
                                 const A2aRoute* route, float* out_scales) {
  GenericPath& g = cuda ? gen_cuda_ : gen_cpu_;
  const bool fused = fused_sharded(cuda);
  if (fused) fused_->check_status();
  const bool routed = route != nullptr && (route->in_index != nullptr || route->out_index != nullptr);
  if (nodes() > 1) {
    // every rank evaluates the same conditions, so every rank refuses and none is left waiting
    if (world_ > kA2aMaxWorld)
      throw std::runtime_error("cgx: the compressed all_to_all supports at most " + std::to_string(kA2aMaxWorld) +
                               " ranks, got " + std::to_string(world_));
    if (!cuda) throw std::runtime_error("cgx: the compressed all_to_all over several nodes needs device memory");
    check_all_to_all(in, out, in_counts, out_counts, dtype, bits, codec, bucket, rank_, world_, route, out_scales);
    if (routed) throw std::logic_error("cgx: a routed all_to_all reached a path that does not route rows");
    if (codec != kMaxMin && !fp8_sr(codec) && rng_in.stochastic)
      throw std::invalid_argument("cgx all_to_all: the FP8 codecs round to nearest only");
    if (!g.world_comm) throw std::runtime_error("cgx: the compressed all_to_all over several nodes has no world communicator");
    if (!fused && local_size_ > 1 && !g.intra)
      throw std::runtime_error("cgx: the compressed all_to_all has no intra-node reducer");
    a2a_nodes(in, out, in_counts, out_counts, dtype, bits, codec, bucket, rng_in, stream, route, out_scales);
    return;
  }
  check_all_to_all(in, out, in_counts, out_counts, dtype, bits, codec, bucket, rank_, world_, route, out_scales);
  if (routed && !routes_in_kernel(cuda, dtype, bits, bucket, route->row))
    throw std::logic_error("cgx: a routed all_to_all reached a path that does not route rows");
  if (!fused && world_ > 1 && !g.intra) throw std::runtime_error("cgx: the compressed all_to_all has no intra-node reducer");
  uint64_t total = 0;
  for (uint64_t n : in_counts) total += n;
  NvtxRange range("cgx:all_to_all_cuda", total);
  ++call_seq_;
  ++stats_.calls;
  RngParams rng = rng_in;
  rng.seq = call_seq_ << 4;
  stats_.elements += total;
  a2a_node(cuda, in, out, in_counts, out_counts, dtype, bits, codec, bucket, rng, stream, route, out_scales, 0);
}

void AllreduceEngine::a2a_node(bool cuda, const void* in, void* out, const std::vector<uint64_t>& in_counts,
                               const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec,
                               uint32_t bucket, const RngParams& rng, cudaStream_t stream, const A2aRoute* route,
                               float* out_scales, int rank_base) {
  GenericPath& g = cuda ? gen_cuda_ : gen_cpu_;
  const int L = local_size_, lr = local_rank();
  if (fused_sharded(cuda)) {
    const FusedSra::A2aCounts n = fused_->all_to_all(in, out, in_counts, out_counts, dtype, bits, codec, bucket, rng,
                                                     stream, route, out_scales, rank_base);
    stats_.kernel_launches += n.launches;
    stats_.wire_bytes += n.wire_bytes;
    stats_.raw_bytes += n.raw_bytes;
    return;
  }
  if (L == 1 && out_scales != nullptr) {
    if (!g.ops) throw std::runtime_error("cgx: the compressed all_to_all has no block backend");
    if (!g.self) {
      g.self_comm = std::make_unique<SelfCommunicator>(cuda);
      g.self = make_reducer(ReductionType::kSRA, g.self_comm.get(), g.ops.get());
    }
    g.self->all_to_all(in, out, in_counts, out_counts, dtype, bits, codec, bucket, rng, stream, out_scales);
    return;
  }
  if (L == 1) {
    const size_t bytes = (size_t)in_counts[0] * (size_t)dtype_size(dtype);
    if (bytes == 0) return;
    if (cuda)
      cuda_check(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream), "all_to_all copy");
    else
      std::memcpy(out, in, bytes);
    return;
  }
  const uint64_t before = g.intra->bytes_sent();
  g.intra->all_to_all(in, out, in_counts, out_counts, dtype, bits, codec, bucket, rng, stream, out_scales, rank_base);
  stats_.wire_bytes += g.intra->bytes_sent() - before;
  for (int q = 0; q < L; ++q)
    if (q != lr) stats_.raw_bytes += in_counts[q] * (uint64_t)dtype_size(dtype);
}

uint64_t a2a_remote_params(A2aRemoteParams& p, const std::vector<uint64_t>& counts, int rank, int L, int dtype,
                           int bits, WireCodec codec, uint32_t bucket, std::vector<uint64_t>* wire,
                           std::vector<uint64_t>* region) {
  const int W = (int)counts.size();
  const int es = dtype_size(dtype);
  const bool raw = bits >= kRawBits;
  std::memset(&p, 0, sizeof(p));
  p.dtype = dtype;
  p.bits = bits;
  p.codec = codec;
  p.bucket = bucket;
  p.rank = rank;
  wire->assign(W, 0);
  region->assign(W, 0);
  uint64_t off = 0, at = 0;
  for (int q = 0; q < W; off += counts[q], ++q) {
    if (q / L == rank / L || counts[q] == 0) continue;
    const A2aGeom g = a2a_geom((uint32_t)counts[q], bits, bucket, es);
    (*wire)[q] = raw ? counts[q] * (uint64_t)es : a2a_chunk_wire(g);
    if (raw) continue;
    (*region)[q] = at;
    const int i = p.nchunks++;
    p.peer[i] = q;
    p.cnt[i] = (uint32_t)counts[q];
    p.elem_off[i] = off;
    p.wire_off[i] = at;
    p.item_first[i + 1] = p.item_first[i] + a2a_chunk_items(g);
    at += a2a_region_bytes((*wire)[q]);
  }
  return at;
}

// Several nodes (DESIGN §2.13f). The chunks for and from the ranks of my node are contiguous in
// `in` and `out`: that sub-range is a one-node all-to-all among my node's ranks. Every other chunk
// is packed into one send buffer (one 256-byte aligned region per destination, its records exactly
// Reducer::all_to_all's), exchanged over the world communicator after the node-local stage and unpacked; at bits >= 32 the
// chunks travel as their bytes, straight from `in` into `out`. Streams and the sequence number are
// those of a one-node call of W ranks.
void AllreduceEngine::a2a_nodes(const void* in, void* out, const std::vector<uint64_t>& in_counts,
                                const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec,
                                uint32_t bucket, const RngParams& rng_in, cudaStream_t stream, const A2aRoute* route,
                                float* out_scales) {
  GenericPath& g = gen_cuda_;
  const int W = world_, L = local_size_, n0 = node() * L;
  const size_t es = (size_t)dtype_size(dtype), oes = out_scales != nullptr ? 1 : es;
  const bool raw = bits >= kRawBits;
  uint64_t total = 0;
  for (uint64_t n : in_counts) total += n;
  NvtxRange range("cgx:all_to_all_cuda", total);
  ++call_seq_;
  ++stats_.calls;
  RngParams rng = rng_in;
  rng.seq = call_seq_ << 4;
  stats_.elements += total;
  std::vector<uint64_t> io(W + 1, 0), oo(W + 1, 0);
  for (int q = 0; q < W; ++q) {
    io[q + 1] = io[q] + in_counts[q];
    oo[q + 1] = oo[q] + out_counts[q];
  }
  // the remote chunks' records and their regions
  auto pk = std::make_unique<A2aRemoteParams>();
  auto up = std::make_unique<A2aRemoteParams>();
  std::vector<uint64_t> sw, rw, so, ro;
  const uint64_t send_bytes = a2a_remote_params(*pk, in_counts, rank_, L, dtype, bits, codec, bucket, &sw, &so);
  const uint64_t recv_bytes = a2a_remote_params(*up, out_counts, rank_, L, dtype, bits, codec, bucket, &rw, &ro);
  pk->rng = make_rng_key(rng, rank_, 0);
  up->out_scales = out_scales;
  auto buffer = [&](GenericPath::Buf& b, uint64_t bytes) -> uint8_t* {
    if (b.cap < bytes) {
      if (b.p) {
        cuda_check(cudaStreamSynchronize(stream), "all_to_all scratch");  // an earlier call may still use it
        g.ops->release(b.p);
      }
      b.cap = std::max<size_t>(bytes, b.cap * 2);
      b.p = g.ops->alloc(b.cap);
    }
    return static_cast<uint8_t*>(b.p);
  };
  uint8_t* sendb = raw ? nullptr : buffer(g.a2a_send, send_bytes + 16);
  uint8_t* recvb = raw ? nullptr : buffer(g.a2a_recv, recv_bytes + 16);
  const uint8_t* src = static_cast<const uint8_t*>(in);
  uint8_t* dst = static_cast<uint8_t*>(out);
  if (pk->nchunks > 0) {
    pk->in = in;
    pk->out = sendb;
    cuda_check(launch_a2a_pack(*pk, stream), "launch_a2a_pack");
  }
  static const std::vector<LayerSpec> kNoLayers;
  std::vector<P2POp> x;
  for (int q = 0; q < W; ++q) {
    if (sw[q]) x.push_back({true, raw ? const_cast<uint8_t*>(src + io[q] * es) : sendb + so[q], sw[q], q});
    if (rw[q]) x.push_back({false, raw ? dst + oo[q] * es : recvb + ro[q], rw[q], q});
    stats_.wire_bytes += sw[q];
    stats_.raw_bytes += in_counts[q] * es * (sw[q] != 0);
  }
  observe(EngineStage::kA2aIntra, &kNoLayers, rng, 1.0f);
  {
    NvtxRange r1("cgx:intra_node", (uint64_t)node());
    const std::vector<uint64_t> ic(in_counts.begin() + n0, in_counts.begin() + n0 + L);
    const std::vector<uint64_t> oc(out_counts.begin() + n0, out_counts.begin() + n0 + L);
    a2a_node(true, src + io[n0] * es, dst + oo[n0] * oes, ic, oc, dtype, bits, codec, bucket, rng, stream, route,
             out_scales != nullptr ? out_scales + oo[n0] / bucket : nullptr, n0);
  }
  observe(EngineStage::kA2aCross, &kNoLayers, rng, 1.0f);
  {
    NvtxRange r2("cgx:cross_node", (uint64_t)nodes());
    g.world_comm->exchange(x, stream);
  }
  if (up->nchunks > 0) {
    up->in = recvb;
    up->out = out;
    cuda_check(launch_a2a_unpack(*up, stream), "launch_a2a_unpack");
  }
}

bool AllreduceEngine::routes_in_kernel(bool cuda, int dtype, int bits, uint32_t bucket, uint64_t row) const {
  return nodes() == 1 && fused_sharded(cuda) && row < (1ull << 32) && a2a_rows_fit((uint32_t)row, bits, bucket, dtype_size(dtype));
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
                                  bool skip_incomplete, float prescale, RngParams rng, cudaStream_t stream,
                                  WireCodec codec) {
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
          launch_fused(Launch{dp, true, rng.seq & 15u, 0u}, data, prescale, rng, stream, codec, &group);
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
      launch_fused(Launch{dp, false, rng.seq & 15u, sub++}, data, prescale, rng, stream, codec, &gl);
    }
    return;
  }
  if (g.intra) {
    const uint64_t before = g.intra->bytes_sent();
    observe(EngineStage::kGenericIntra, &group, rng, prescale);
    g.intra->allreduce(data, dtype, group, skip_incomplete, prescale, rng, stream, codec);
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
  const bool multi_node = nodes() > 1;
  const WireCodec codec = (WireCodec)env.codec;
  if (codec != kMaxMin) {  // checked before anything is counted or sent
    if (env.stochastic && !fp8_sr(codec))
      throw std::invalid_argument("cgx allreduce: the FP8 formats round to nearest only");
    for (const LayerSpec& l : layers)
      if (l.bits != 8 && l.bits < kRawBits)
        throw std::invalid_argument("cgx allreduce: an FP8 format needs layers of bits 8 or 32, got " +
                                    std::to_string(l.bits));
    if (cfg_.inner_reduction == ReductionType::kAllToAll ||
        (multi_node && cfg_.cross_reduction == ReductionType::kAllToAll))
      throw std::invalid_argument(kAllToAllNoFp8);
  }
  ++call_seq_;
  ++stats_.calls;
  RngParams rng;
  rng.seed = env.seed;
  rng.stochastic = env.stochastic;
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
      intra_stage(cuda, data, dtype, intra_layers, env.skip_incomplete, prescale, rng, stream, codec);
    }
    if (!multi_node) continue;
    NvtxRange r2("cgx:cross_node", (uint64_t)group.size());
    // ---- stage 2: across nodes (reference: mpi_allreduce_operations.cc:161-183)
    RngParams crng = rng;
    crng.seq = rng.seq ^ 0x40000000u;
    const float cross_scale = (local_size_ > 1) ? 1.0f : prescale;
    if (cfg_.intra_broadcast && local_size_ > 1) {
      if (local_rank() == 0) {
        observe(EngineStage::kCross, &group, crng, cross_scale);
        g.cross->allreduce(data, dtype, group, env.skip_incomplete, cross_scale, crng, stream, codec);
      }
      // leaders hand the result to the rest of their node: packed when the intra-node stage
      // compresses (reference: Reducer::Broadcast with do_compression && intra_compress_,
      // mpi_allreduce_operations.cc:171-176, reducer.cc:96-160), raw bytes of the span otherwise
      bool any_compressed = false;
      for (const LayerSpec& l : group) any_compressed = any_compressed || l.bits < kRawBits;
      if (g.intra && cfg_.intra_compress && any_compressed) {
        RngParams brng = rng;
        brng.seq = rng.seq ^ 0x20000000u;
        const uint64_t before = g.intra->bytes_sent();
        observe(EngineStage::kBcastCompressed, &group, brng, 1.0f);
        g.intra->broadcast_compressed(data, dtype, group, env.skip_incomplete, 0, brng, stream, codec);
        stats_.wire_bytes += g.intra->bytes_sent() - before;
      } else {
        uint64_t lo = ~0ull, hi = 0;
        for (const LayerSpec& l : group) {
          lo = std::min<uint64_t>(lo, l.elem_off);
          hi = std::max<uint64_t>(hi, l.elem_off + l.numel);
        }
        if (hi > lo && g.intra) {
          observe(EngineStage::kBcastRaw, &group, rng, 1.0f);
          g.intra->broadcast(static_cast<uint8_t*>(data) + lo * elsize, (size_t)(hi - lo) * elsize, 0, stream);
        }
      }
    } else {
      observe(EngineStage::kCross, &group, crng, cross_scale);
      g.cross->allreduce(data, dtype, group, env.skip_incomplete, cross_scale, crng, stream, codec);
    }
  }
}

}  // namespace cgx

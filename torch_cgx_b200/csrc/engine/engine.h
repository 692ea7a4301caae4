// Allreduce orchestration: layer extraction, compress / no-compress decision,
// tensor-fusion chunking, dispatch to a reducer.
//
// Reference: MPIAllReduce_Operation (/root/reference/src/mpi_allreduce_operations
// .h:34-85, .cc:117-287). Differences by design: compressed and uncompressed
// layers of a bucket go through the SAME kernel launch (raw blocks) instead of
// two reducer passes; the plan is cached per layout; nothing here touches MPI.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <memory>
#include <mutex>
#include <optional>
#include <vector>

#include "../comm/symmetric_heap.h"
#include "../common/config.h"
#include "../common/layers.h"
#include "../comm/communicator.h"
#include "../kernels/launch.h"
#include "../reduce/block_backend.h"
#include "../reduce/fused_sra.h"
#include "../reduce/reducers.h"

namespace cgx {

struct EngineStats {
  uint64_t calls = 0;            // allreduce and compressed reduce-scatter / all-gather calls, together
  uint64_t kernel_launches = 0;  // fused kernel launches
  uint64_t elements = 0;
  uint64_t wire_bytes = 0;       // bytes this rank pushed over NVLink (both phases)
  uint64_t raw_bytes = 0;        // bytes an uncompressed SRA would have pushed
};

// Split a layer list into groups whose raw size fits `fusion_bytes`
// (Horovod-style tensor fusion threshold; a single layer larger than the
// threshold is sliced at bucket boundaries). Unlike the reference
// (mpi_allreduce_operations.cc:201-227, SURVEY.md §2.8 #2) no trailing group is
// ever dropped.
std::vector<std::vector<LayerSpec>> split_for_fusion(const std::vector<LayerSpec>& layers, int elsize,
                                                     int64_t fusion_bytes);

// One stage of an allreduce or of a sharded collective as the engine issues it (EngineObserver::stage).
// kRs / kAg are fused launches (one per window), kGenericRs / kGenericAg the generic intra-node
// reducer, kCrossRs / kCrossAg the cross-node stage of a sharded call. An all-to-all over several
// nodes issues kA2aIntra (the node's own chunks) and then kA2aCross (the exchange of the packed
// remote chunks); one node issues none.
struct EngineStage {
  enum Kind {
    kOneshot, kSra, kGenericIntra, kCross, kBcastCompressed, kBcastRaw,
    kRs, kAg, kGenericRs, kGenericAg, kCrossRs, kCrossAg, kA2aCross, kA2aIntra
  };
  Kind kind;
  // the stage's layer table (a sharded stage: one shard's, or a fused launch's window of it); null
  // for a fused launch of the bucket fast path
  const std::vector<LayerSpec>* layers;
  const DevicePlan* dp;                  // the plan of a fused launch (kOneshot / kSra / kRs / kAg), else null
  RngParams rng;                         // the sequence number the stage runs with
  float scale;                           // prescale of a reduction stage, 1 for a broadcast or an all-gather
  bool sharded() const { return kind >= kRs && kind <= kCrossAg; }
  bool a2a() const { return kind >= kA2aCross; }
};

// Test seam: sees every stage an engine issues. Production engines have none (one branch per stage).
class EngineObserver {
 public:
  virtual ~EngineObserver() = default;
  // right before a fused kernel launch, slow and fast path alike
  virtual void before_fused_launch(const DevicePlan& dp, cudaStream_t stream) = 0;
  virtual void stage(const EngineStage& s) = 0;
};

// Reducers of one memory kind (host or device): the generic intra-node and
// cross-node stages of the hierarchical allreduce.
struct GenericPath {
  std::unique_ptr<BlockBackend> ops;
  std::unique_ptr<Communicator> intra_comm;  // ranks of my node (null if the node has one rank)
  std::unique_ptr<Communicator> cross_comm;  // ranks with my local rank on the other nodes (null if one node)
  std::unique_ptr<Reducer> intra;
  std::unique_ptr<Reducer> cross;
  // world 1: a reducer over a one-rank communicator, made on first use, that encodes the all-to-all's
  // codes output (nothing is exchanged)
  std::unique_ptr<Communicator> self_comm;
  std::unique_ptr<Reducer> self;
  // all the world's ranks: the exchange of the all-to-all's cross-node chunks (null on one node)
  std::unique_ptr<Communicator> world_comm;
  // grow-only send and receive buffers of that exchange
  struct Buf {
    void* p = nullptr;
    size_t cap = 0;
  };
  Buf a2a_send, a2a_recv;
};

// The parameters of the cross-node all-to-all's pack (counts: this rank's input counts) or unpack
// (its output counts) launch for world rank `rank` with nodes of L ranks: every chunk for or from a
// rank of another node, in rank order, its records in a 256-byte aligned region of one buffer.
// wire[q] receives chunk q's record bytes (its bytes at bits >= 32, which launch nothing), 0 for my
// node's ranks; region[q] its region's offset. Returns the buffer's bytes.
uint64_t a2a_remote_params(A2aRemoteParams& p, const std::vector<uint64_t>& counts, int rank, int L, int dtype,
                           int bits, WireCodec codec, uint32_t bucket, std::vector<uint64_t>* wire,
                           std::vector<uint64_t>* region);

class AllreduceEngine {
 public:
  AllreduceEngine(int rank, int world, const EngineConfig& cfg);
  ~AllreduceEngine();

  // Topology: `local_size` consecutive ranks form a node (reference: MPIContext's
  // shared-memory split, /root/reference/src/common/mpi_context.cc:25-35;
  // overridable with CGX_LOCAL_SIZE to simulate several nodes on one box).
  void set_topology(int local_size);
  int local_size() const { return local_size_; }
  int local_rank() const { return rank_ % local_size_; }
  int node() const { return rank_ / local_size_; }
  int nodes() const { return world_ / local_size_; }

  // Install the generic reducers for host (cuda == false) or device memory.
  // Communicators may be null where the corresponding group has a single rank.
  void attach_generic(bool cuda, std::unique_ptr<Communicator> intra, std::unique_ptr<Communicator> cross);
  bool has_generic(bool cuda) const { return (cuda ? gen_cuda_ : gen_cpu_).ops != nullptr; }
  // The communicator of all the world's ranks (rank() the world rank) that carries the cross-node
  // chunks of a compressed all-to-all over several nodes; needs attach_generic(cuda) first.
  void attach_world(bool cuda, std::unique_ptr<Communicator> world);

  // In-place SUM/AVG allreduce of a host buffer through the generic reducers.
  void allreduce_cpu(void* data, int dtype, int64_t numel, bool average, int explicit_bucket);
  // The same in two steps, for callers that run the reduction on another thread: the environment
  // and the layer table are read on the CALLING thread (they may change right after the call
  // returns, e.g. the `compression()` context manager), the work runs later.
  struct CpuCall {
    CompressionEnv env;
    std::vector<LayerSpec> layers;
  };
  CpuCall prepare_cpu(int64_t numel, int explicit_bucket) const;
  void allreduce_cpu_prepared(void* data, int dtype, const CpuCall& call, bool average);

  const EngineConfig& config() const { return cfg_; }
  int rank() const { return rank_; }
  int world() const { return world_; }

  // slot size the symmetric heap needs for this config
  static size_t required_slot_bytes(const EngineConfig& cfg, int world);
  static size_t required_oneshot_slot_bytes(const EngineConfig& cfg);

  // takes ownership of a connected heap and enables the fused P2P path
  void attach_heap(std::unique_ptr<SymmetricHeap> heap, int lanes);
  bool has_p2p() const { return fused_ != nullptr; }
  SymmetricHeap* heap() { return heap_.get(); }
  FusedSra* fused() { return fused_.get(); }

  // In-place SUM (or AVG) allreduce of a CUDA buffer on `stream`.
  //  explicit_bucket: DDP bucket index if the caller knows it, else -1.
  //  overlapped: the call runs concurrently with compute (DDP hook) -> use at most
  //  cfg.overlap_lanes CTAs instead of the whole GPU.
  //  codec: the wire format of the 8-bit layers, replacing CGX_COMPRESSION_FORMAT's when given.
  // With an FP8 format (CompressionEnv::codec) every layer must have bits 8 or 32 and rounding is to
  // nearest; every compressed stage (node-local, cross-node, the leaders' compressed broadcast) uses
  // it. std::invalid_argument otherwise, before any stage runs.
  void allreduce_cuda(void* data, int dtype, int64_t numel, bool average, int explicit_bucket,
                      cudaStream_t stream, bool overlapped = false, std::optional<WireCodec> codec = std::nullopt);
  // Same, with an explicit layer list (offsets relative to `data`).
  void allreduce_cuda_layers(void* data, int dtype, const std::vector<LayerSpec>& layers, bool average,
                             const CompressionEnv& env, cudaStream_t stream, bool overlapped = false);

  // Compressed reduce-scatter or all-gather of device (cuda) or host buffers on `stream` with shards
  // of S = shard_numel elements: the reduce-scatter's `in` holds world * S elements and `out`
  // receives this rank's shard; the all-gather's `in` is this rank's shard and `out` receives
  // world * S, every shard (this rank's included) one quantization round trip (average and
  // skip_incomplete false). `shard_layers` is one shard's table (sharded_table).
  // One node: the fused kernel (FusedSra::sharded) on the P2P transport, else the generic intra-node
  // reducer. Several nodes: two stages (DESIGN §2.9b), the node-local one as on one node, the other
  // through the cross-node reducer; `staging` then holds sharded_staging_numel(S) elements of the
  // dtype for the node partials / the gathered shards. Host memory runs the generic reducers only.
  // Adds to the same counters as the allreduce. An FP8 `codec` (layers of bits 8 or 32) is the wire
  // format of every compressed stage, node-local and cross-node (FusedSra::sharded).
  // `out_scales` selects the all-gather's codes output (check_sharded_buffers, FusedSra::sharded); it
  // runs on one node only: with several nodes every rank throws the same std::runtime_error before
  // anything runs.
  void sharded(bool cuda, ShardedOp op, const void* in, void* out, void* staging, int dtype, int64_t shard_numel,
               const std::vector<LayerSpec>& shard_layers, bool average, bool skip_incomplete,
               const RngParams& rng_in, cudaStream_t stream, bool overlapped, WireCodec codec = kMaxMin,
               float* out_scales = nullptr);
  // The table of one S-element shard: `layers` when given, else one layer of S elements with `bits`
  // / `bucket`, raw unless S exceeds CGX_COMPRESSION_MINIMAL_SIZE.
  std::vector<LayerSpec> sharded_table(int64_t shard_numel, std::vector<LayerSpec> layers, int bits,
                                       int bucket) const;
  // elements of the staging buffer sharded() needs: N * S with several nodes of several ranks, else 0
  int64_t sharded_staging_numel(int64_t shard_numel) const {
    return (nodes() > 1 && local_size_ > 1) ? (int64_t)nodes() * shard_numel : 0;
  }
  // builds and uploads every fused plan a sharded() call with this table launches, without launching
  void prepare_sharded(ShardedOp op, const std::vector<LayerSpec>& shard_layers, int dtype, bool skip_incomplete,
                       cudaStream_t stream);

  // Compressed all-to-all of device (cuda) or host buffers on `stream` (FusedSra::all_to_all for
  // the arguments): the fused kernel on the P2P transport, else the generic intra-node reducer.
  // A `route` with an index needs routes_in_kernel(); callers compose index_select / index_copy_
  // around a plain call otherwise. `out_scales` selects the codes output (FusedSra::all_to_all); at
  // world 1 without a heap the chunk is then encoded by the generic reducer's path, not copied.
  // Several nodes (DESIGN §2.13f; device memory, at most kA2aMaxWorld ranks, no route): one launch
  // packs every chunk for another node (launch_a2a_pack), the node's own chunks run the one-node path
  // above on the node's sub-range with world-rank streams, one grouped exchange over the world
  // communicator moves the records, and one launch unpacks the received records. Every chunk is
  // quantized once by its sender and decoded once by its receiver: the result is the one-node
  // all-to-all of W ranks, bit for bit.
  void all_to_all(bool cuda, const void* in, void* out, const std::vector<uint64_t>& in_counts,
                  const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec, uint32_t bucket,
                  const RngParams& rng_in, cudaStream_t stream, const A2aRoute* route = nullptr,
                  float* out_scales = nullptr);
  // whether a routed all-to-all of rows of `row` elements runs inside the fused kernel: the P2P
  // transport with a heap, and rows that hold whole quantization items (a2a_rows_fit)
  bool routes_in_kernel(bool cuda, int dtype, int bits, uint32_t bucket, uint64_t row) const;

  void check_health();
  void set_observer(EngineObserver* o) { observer_ = o; }
  const EngineStats& stats() const { return stats_; }
  void reset_stats() { stats_ = EngineStats(); }

 private:
  void run_layers(bool cuda, void* data, int dtype, std::vector<LayerSpec> layers, bool average,
                  const CompressionEnv& env, cudaStream_t stream);
  void intra_stage(bool cuda, void* data, int dtype, const std::vector<LayerSpec>& group, bool skip_incomplete,
                   float prescale, RngParams rng, cudaStream_t stream, WireCodec codec);
  // the node-local stage of a sharded call over the local ranks: fused kernel or generic reducer
  void sharded_intra(bool cuda, ShardedOp op, const void* in, void* out, int dtype, uint64_t S,
                     const std::vector<LayerSpec>& table, bool skip_incomplete, float prescale, const RngParams& rng,
                     cudaStream_t stream, bool overlapped, WireCodec codec, float* out_scales = nullptr);
  bool fused_sharded(bool cuda) const { return cuda && fused_ && cfg_.inner_comm == CommType::kP2P; }
  // the all-to-all among the ranks of my node: counts and buffers of the node's sub-range, the
  // streams of world ranks rank_base + local rank
  void a2a_node(bool cuda, const void* in, void* out, const std::vector<uint64_t>& in_counts,
                const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec, uint32_t bucket,
                const RngParams& rng, cudaStream_t stream, const A2aRoute* route, float* out_scales, int rank_base);
  void a2a_nodes(const void* in, void* out, const std::vector<uint64_t>& in_counts,
                 const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec, uint32_t bucket,
                 const RngParams& rng_in, cudaStream_t stream, const A2aRoute* route, float* out_scales);
  // the node-local stage's table: raw in a multi-node all-gather, and in a multi-node
  // reduce-scatter without CGX_INTRA_COMPRESS
  std::vector<LayerSpec> sharded_intra_table(ShardedOp op, std::vector<LayerSpec> table) const;

  // Fast path for registered DDP buckets: once a bucket's plans are known (and nothing that
  // influences them changed) a call is just "launch these kernels" -- no layer extraction,
  // no fusion split, no plan hashing on the host.
  struct Launch {
    const DevicePlan* dp;
    bool oneshot;
    uint32_t rng_group;  // fusion group of this launch (low bits of the call's RNG sequence)
    uint32_t rng_sub;    // piece of the group (low bits of the launch's RNG sequence)
  };
  struct BucketFast {
    uint64_t registry_version = 0;
    uint64_t plan_generation = 0;
    int64_t numel = -1;
    int dtype = -1;
    int env_bits = 0, env_bucket = 0, env_codec = 0;
    bool skip_incomplete = false;
    bool overlapped = false;
    std::vector<Launch> launches;
  };
  std::vector<BucketFast> fast_;
  std::vector<Launch>* recording_ = nullptr;
  void launch_fused(const Launch& l, void* data, float prescale, RngParams rng, cudaStream_t stream,
                    WireCodec codec, const std::vector<LayerSpec>* layers = nullptr);
  void observe(EngineStage::Kind kind, const std::vector<LayerSpec>* layers, const RngParams& rng, float scale) {
    if (observer_) observer_->stage(EngineStage{kind, layers, nullptr, rng, scale});
  }

  int rank_, world_;
  int local_size_;
  EngineConfig cfg_;
  GenericPath gen_cuda_, gen_cpu_;
  std::unique_ptr<SymmetricHeap> heap_;
  std::unique_ptr<FusedSra> fused_;
  std::mutex cpu_mu_;
  uint32_t call_seq_ = 0;
  int lane_cap_ = 0;  // lane cap of the call being issued (0 = none)
  EngineStats stats_;
  EngineObserver* observer_ = nullptr;
};

}  // namespace cgx

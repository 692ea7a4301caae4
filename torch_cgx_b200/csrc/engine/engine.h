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
#include <vector>

#include "../comm/symmetric_heap.h"
#include "../common/config.h"
#include "../common/layers.h"
#include "../comm/communicator.h"
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

// Reducers of one memory kind (host or device): the generic intra-node and
// cross-node stages of the hierarchical allreduce.
struct GenericPath {
  std::unique_ptr<BlockBackend> ops;
  std::unique_ptr<Communicator> intra_comm;  // ranks of my node (null if the node has one rank)
  std::unique_ptr<Communicator> cross_comm;  // ranks with my local rank on the other nodes (null if one node)
  std::unique_ptr<Reducer> intra;
  std::unique_ptr<Reducer> cross;
};

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
  void allreduce_cuda(void* data, int dtype, int64_t numel, bool average, int explicit_bucket,
                      cudaStream_t stream, bool overlapped = false);
  // Same, with an explicit layer list (offsets relative to `data`).
  void allreduce_cuda_layers(void* data, int dtype, const std::vector<LayerSpec>& layers, bool average,
                             const CompressionEnv& env, cudaStream_t stream, bool overlapped = false);

  // Compressed reduce-scatter or all-gather of CUDA buffers on `stream` (FusedSra::sharded) with
  // shards of S = shard_numel elements: the reduce-scatter's `in` holds world * S elements and
  // `out` receives this rank's shard; the all-gather's `in` is this rank's shard and `out`
  // receives world * S, every shard (this rank's included) one quantization round trip (average
  // and skip_incomplete false). An empty `shard_layers` means one layer of S elements with
  // `bits` / `bucket`, raw unless S exceeds CGX_COMPRESSION_MINIMAL_SIZE. Single node, P2P
  // transport only; adds to the same counters as the allreduce.
  void sharded_cuda(ShardedOp op, const void* in, void* out, int dtype, int64_t shard_numel,
                    std::vector<LayerSpec> shard_layers, bool average, int bits, int bucket, bool skip_incomplete,
                    const RngParams& rng_in, cudaStream_t stream, bool overlapped);

  void check_health();
  const EngineStats& stats() const { return stats_; }
  void reset_stats() { stats_ = EngineStats(); }

 private:
  void run_layers(bool cuda, void* data, int dtype, std::vector<LayerSpec> layers, bool average,
                  const CompressionEnv& env, cudaStream_t stream);
  void intra_stage(bool cuda, void* data, int dtype, const std::vector<LayerSpec>& group, bool skip_incomplete,
                   float prescale, RngParams rng, cudaStream_t stream);

  // Fast path for registered DDP buckets: once a bucket's plans are known (and nothing that
  // influences them changed) a call is just "launch these kernels" -- no layer extraction,
  // no fusion split, no plan hashing on the host.
  struct Launch {
    const DevicePlan* dp;
    bool oneshot;
    uint32_t rng_sub;  // low bits of the RNG sequence used for this launch
  };
  struct BucketFast {
    uint64_t registry_version = 0;
    uint64_t plan_generation = 0;
    int64_t numel = -1;
    int dtype = -1;
    int env_bits = 0, env_bucket = 0;
    bool skip_incomplete = false;
    bool overlapped = false;
    std::vector<Launch> launches;
  };
  std::vector<BucketFast> fast_;
  std::vector<Launch>* recording_ = nullptr;
  void launch_fused(const Launch& l, void* data, float prescale, RngParams rng, cudaStream_t stream);

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
};

}  // namespace cgx

// Host driver of the fused P2P Scatter-Reduce-AllGather kernel: plan cache,
// epoch counter, launch. One instance per (process group, device).
// Reference role: MPI_Allreduce_ScatterReduceAllgather::AllreduceCompressed /
// AllreduceUncompressed (/root/reference/src/common/scatter_reduce_allgather.cc
// :94-202, :308-413) and NCCL_Reduce (/root/reference/src/common/nccl_reduce.cc
// :103-198) -- collapsed into a single kernel launch per call.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../comm/symmetric_heap.h"
#include "../common/plan.h"
#include "../common/sra_sim.h"

namespace cgx {

struct DevicePlan {
  Plan plan;
  WarpItem* d_items = nullptr;       // flattened warp work list (device)
  uint32_t* d_item_first = nullptr;  // [world * lanes + 1]
  bool multicast_ok = false;         // every compressed item has a width multimem.st can carry (2/4/8)
};

// The two sharded collectives. Both move S-element shards through one table and the same windows;
// the reduce-scatter reads W * S elements and writes the shard, the all-gather the other way round.
enum class ShardedOp { kReduceScatter, kAllGather };
inline const char* op_name(ShardedOp op) { return op == ShardedOp::kReduceScatter ? "reduce_scatter" : "all_gather"; }
inline const char* op_title(ShardedOp op) { return op == ShardedOp::kReduceScatter ? "reduce-scatter" : "all-gather"; }

// S: end of a shard table, which must tile [0, S) in order
inline uint64_t shard_elems(const std::vector<LayerSpec>& layers) {
  uint64_t end = 0;
  for (const LayerSpec& l : layers) {
    if (l.elem_off != end)
      throw std::invalid_argument("cgx reduce_scatter: the shard layers must tile [0, S) in order, without gaps");
    end += l.numel;
  }
  return end;
}

// a shard table's plan table: W copies at stride S, copy c = chunk c
inline std::vector<LayerSpec> replicate(const std::vector<LayerSpec>& shard, int world, uint64_t S) {
  std::vector<LayerSpec> out;
  out.reserve(shard.size() * (size_t)world);
  for (int c = 0; c < world; ++c)
    for (LayerSpec l : shard) {
      l.elem_off += (uint64_t)c * S;
      out.push_back(l);
    }
  return out;
}

// The windows of a reduce-scatter: the shard's layer table (offsets from the shard start, tiling
// [0, S) in order; std::invalid_argument otherwise) cut by split_for_fusion into shard-relative
// tables whose plans -- the window replicated opt.world times at stride S -- fit `slot_bytes` per
// chunk. Cuts fall on bucket boundaries (for buckets above kMaxBlockElems on multiples of both
// sizes), so the result of the operation does not depend on the windows.
std::vector<std::vector<LayerSpec>> reduce_scatter_windows(const std::vector<LayerSpec>& shard_layers,
                                                           const PlanOptions& opt, uint32_t slot_bytes);

class FusedSra {
 public:
  FusedSra(SymmetricHeap* heap, int max_lanes, int64_t timeout_ms, uint32_t min_lane_elems);
  ~FusedSra();

  int rank() const { return heap_->rank(); }
  int world() const { return heap_->world(); }
  int max_lanes() const { return max_lanes_; }

  // Build (or fetch) the plan for `layers`; returns nullptr if its largest
  // chunk does not fit the heap's slots (caller must split the call).
  //  max_lanes > 0 caps the number of lanes (CTAs) below the group's maximum: calls that overlap
  //  with compute (DDP buckets during backward) leave most SMs to the model.
  const DevicePlan* prepare(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                            cudaStream_t stream, int max_lanes = 0);

  // In-place allreduce of `data` over the layers of `dp`. Stream-ordered, no
  // host synchronisation. Every rank must call this the same number of times
  // in the same order (epoch counter).
  void run(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream);

  // One-shot variant (single signalling hop, for latency-bound messages): plan over the WHOLE
  // buffer (one chunk); nullptr if its packed image does not fit the heap's one-shot slots.
  const DevicePlan* prepare_oneshot(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                                    cudaStream_t stream, int max_lanes = 0);
  void run_oneshot(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream);

  // A sharded collective over S-element shards; `shard_layers` is the quantization table of ONE
  // shard (offsets from the shard start, tiling [0, S)); every shard uses it, so buckets are counted
  // from each shard's start. The shard buffer is disjoint from the full buffer or exactly its chunk
  // rank(); anything else throws std::invalid_argument.
  //  kReduceScatter (rs_kernel): `in` holds W * S elements, `out` S; this rank receives shard rank():
  //    out = T(prescale * in[r] + sum over peers p of decode(Q(prescale * in_p[r]))).
  //  kAllGather (ag_kernel): `in` holds this rank's shard, `out` W * S: out[q * S + i] =
  //    decode(Q_q(in_q[i])) for every rank q, this rank's own shard included, so every rank's `out`
  //    is the same bytes (bits 32 = copied unchanged). Rounds to nearest unless rng.stochastic;
  //    callers pass skip_incomplete = false and prescale = 1.
  // The shard is cut into windows whose worst-case wire fits one slot (split_for_fusion, cuts on
  // bucket boundaries, so the result does not depend on the slot size) and one kernel is launched
  // per window. Stream-ordered; every rank must issue the same calls in the same order.
  struct RsCounts {
    uint64_t launches = 0, elements = 0, wire_bytes = 0, raw_bytes = 0;  // this rank's share
  };
  RsCounts sharded(ShardedOp op, const std::vector<LayerSpec>& shard_layers, int dtype, bool skip_incomplete,
                   const void* in, void* out, uint64_t S, float prescale, const RngParams& rng, cudaStream_t stream,
                   int max_lanes = 0);
  // builds and uploads the plans of every window without launching anything
  void prepare_sharded(const std::vector<LayerSpec>& shard_layers, int dtype, bool skip_incomplete,
                       cudaStream_t stream, int max_lanes = 0);
  // reduce_scatter_windows for this heap (cached per shard table); the all-gather uses the same
  // windows, since its per-chunk wire is the reduce-scatter's
  const std::vector<std::vector<LayerSpec>>& rs_windows(const std::vector<LayerSpec>& shard_layers, int dtype,
                                                        bool skip_incomplete, int max_lanes);

  // throws std::runtime_error if a kernel reported a timeout / abort (sticky)
  void check_status();
  void clear_status();
  // same, without throwing: empty string when healthy (does not clear the status)
  std::string status_message() const;
  bool uses_multicast() const { return use_mc_; }

  // Tracing: when enabled, the next run() records per-lane phase timestamps
  // (device globaltimer, ns); read_trace() synchronises the device and returns
  // lanes x 8 values: [start, A done, B inputs ready, B done, last C wait, end, -, -].
  void enable_trace(bool on);
  std::vector<uint64_t> read_trace();
  int last_lanes() const { return last_lanes_; }
  uint64_t launches() const { return launches_; }
  // bumped whenever cached DevicePlan pointers become invalid (cache trimmed)
  uint64_t generation() const { return generation_; }
  uint32_t epoch() const { return epoch_; }
  size_t num_plans() const { return cache_.size(); }

 private:
  SymmetricHeap* heap_;
  int max_lanes_;
  uint64_t timeout_ns_;
  uint32_t min_lane_elems_;
  uint32_t epoch_ = 0;  // host mirror of the device-side call counter (DeviceSync)
  uint64_t launches_ = 0;
  bool use_mc_ = false;      // NVLS stores (multimem.st) for phase B / one-shot
  int stages_ = 0;              // CGX_STAGES override of the pipeline depth (0 = automatic)
  int pick_stages(const DevicePlan& dp) const;
  bool use_mc_reduce_ = false;  // NVLS in-switch reduction (multimem.ld_reduce) for raw items
  unsigned long long* d_trace_ = nullptr;
  bool trace_on_ = false;
  int last_lanes_ = 0;
  uint64_t generation_ = 1;
  static constexpr size_t kMaxCachedPlans = 1024;
  const DevicePlan* prepare_impl(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                                 cudaStream_t stream, int plan_world, uint32_t capacity, int max_lanes);
  void launch(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream,
              bool oneshot, void* out = nullptr, uint64_t out_shift = 0, bool gather = false);
  std::unordered_map<uint64_t, std::unique_ptr<DevicePlan>> cache_;
  std::unordered_map<uint64_t, std::vector<std::vector<LayerSpec>>> rs_windows_;
};

}  // namespace cgx

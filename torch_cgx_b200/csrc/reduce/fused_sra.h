// Host driver of the fused P2P Scatter-Reduce-AllGather kernel: plan cache,
// epoch counter, launch. One instance per (process group, device).
// Reference role: MPI_Allreduce_ScatterReduceAllgather::AllreduceCompressed /
// AllreduceUncompressed (/root/reference/src/common/scatter_reduce_allgather.cc
// :94-202, :308-413) and NCCL_Reduce (/root/reference/src/common/nccl_reduce.cc
// :103-198) -- collapsed into a single kernel launch per call.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <functional>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../comm/symmetric_heap.h"
#include "../common/plan.h"
#include "../common/sra_sim.h"
#include "plan_cache.h"

namespace cgx {

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

// The buffers of one rank's sharded call: `shard_layers` tiles [0, S) in order, and the shard buffer
// (the reduce-scatter's `out`, the all-gather's `in`) is disjoint from the full one or exactly its
// chunk `rank` of `world`; with an FP8 `codec` every layer has bits 8 or 32 (raw);
// std::invalid_argument otherwise.
// With `out_scales` (the all-gather's codes output) `out` holds one byte per element and out_scales
// one float per bucket: an FP8 codec, every layer of bits 8 with one bucket B <= kMaxBlockElems
// dividing its size (so every bucket lies inside one shard), and input, codes and scales pairwise
// disjoint.
void check_sharded_buffers(ShardedOp op, const std::vector<LayerSpec>& shard_layers, int dtype, const void* in,
                           const void* out, uint64_t S, int rank, int world, WireCodec codec = kMaxMin,
                           const float* out_scales = nullptr);
// The bucket B of the all-gather's codes output: the scale of the bucket starting at output element
// e is out_scales[e / B]. std::invalid_argument unless `op` is the all-gather, `codec` an FP8 codec
// and the table as check_sharded_buffers requires.
uint32_t codes_bucket(ShardedOp op, const std::vector<LayerSpec>& shard_layers, WireCodec codec);

// The windows of a reduce-scatter: the shard's layer table (offsets from the shard start, tiling
// [0, S) in order; std::invalid_argument otherwise) cut by split_for_fusion into shard-relative
// tables whose plans -- the window replicated opt.world times at stride S -- fit `slot_bytes` per
// chunk. Cuts fall on bucket boundaries (for buckets above kMaxBlockElems on multiples of both
// sizes), so the result of the operation does not depend on the windows.
std::vector<std::vector<LayerSpec>> reduce_scatter_windows(const std::vector<LayerSpec>& shard_layers,
                                                           const PlanOptions& opt, uint32_t slot_bytes);

// The routed form of one rank's all-to-all: the counts describe logical buffers of whole rows of
// `row` elements; row i of the logical send buffer is row in_index[i] of `in` (in_rows rows), row j
// of the logical receive buffer is written to row out_index[j] of `out` (out_rows rows). A nullptr
// index means that side is the logical buffer itself. The index values live on the device and are
// checked by the kernel (kSraBadIndex), not here.
// Weighted top-k combine (DESIGN §2.13d; combine_out != nullptr, with out_index): `out` is the slots
// buffer of out_rows = T * topk rows, slot t * topk + c is choice c of token t, and combine_out
// ([T, row], the input's dtype) receives T(acc), acc = gate[t, 0] * slot 0, then
// fma(gate[t, c], slot c, acc) for c = 1 .. topk - 1. `masks` is zeroed scratch of
// T * (row / a2a_row_span) words for the fused kernel's arrivals.
struct A2aRoute {
  const int64_t* in_index = nullptr;
  const int64_t* out_index = nullptr;
  uint64_t row = 1;
  uint64_t in_rows = 0, out_rows = 0;
  void* combine_out = nullptr;
  const float* gate = nullptr;  // [T, topk] fp32
  uint32_t topk = 0;            // 1..32
  uint32_t* masks = nullptr;
  const float* in_scale = nullptr;  // scaled send: one fp32 per in_index entry (A2aParams::in_scale)
};

// The arguments of one rank's all-to-all (FusedSra::all_to_all, Reducer::all_to_all): a count per
// rank on both sides, bits 1..8 or >= 32 (8 with an FP8 codec), a bucket >= 1, the own chunk the same size on both sides,
// tensors below 2^32 elements and an output that does not overlap the input; with a route, counts
// of whole rows and no overlap of the tensors the indices address; std::invalid_argument otherwise.
// With `out_scales` (the codes output) `out` holds one byte per element and out_scales one float per
// bucket: an FP8 codec, a bucket of at most kMaxBlockElems that divides every count (and the row),
// and codes, scales and input pairwise disjoint. A combine (route->combine_out) needs an out_index
// whose entries are the out_rows = T * topk slots, topk in 1..32, no codes output, and neither
// combine_out nor the gate overlapping the input, or combine_out the slots. A scaled send
// (route->in_scale) needs an in_index, no codes output and no combine, and a scale not overlapping `out`.
void check_all_to_all(const void* in, const void* out, const std::vector<uint64_t>& in_counts,
                      const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec, uint32_t bucket,
                      int rank, int world, const A2aRoute* route = nullptr, const float* out_scales = nullptr);

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
  // in the same order (epoch counter). An FP8 `codec` (common/quant_math.h; a plan of bits 8 or 32,
  // round to nearest, else std::invalid_argument before anything is launched) gives the 8-bit
  // records FP8 codes: the sender encodes prescale * x, the owner adds each decoded value
  // fl(float(code) * unit) with its own rounding, encodes the fp32 sum once and keeps its decoded codes.
  void run(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream,
           WireCodec codec = kMaxMin);

  // One-shot variant (single signalling hop, for latency-bound messages): plan over the WHOLE
  // buffer (one chunk); nullptr if its packed image does not fit the heap's one-shot slots.
  const DevicePlan* prepare_oneshot(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                                    cudaStream_t stream, int max_lanes = 0);
  // An FP8 `codec` as in run(): every rank sums the decoded images from +0.
  void run_oneshot(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream,
                   WireCodec codec = kMaxMin);

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
  // `before_launch`, when set, sees each window's table and plan right before its kernel is launched.
  // An FP8 `codec` (common/quant_math.h; layers of bits 8 or 32, round to nearest) gives the 8-bit
  // records FP8 codes: the sender encodes prescale * x, the reduce-scatter adds each decoded value
  // fl(float(code) * unit) with its own rounding, and the all-gather's owner keeps the decoded codes.
  // With `out_scales` (all-gather, FP8 codec; check_sharded_buffers) `out` receives the codes and
  // out_scales the units of every shard undecoded, the own shard's being the bytes it published
  // (SraParams::out_scales); the wire and the counts are the decoded call's.
  struct RsCounts {
    uint64_t launches = 0, elements = 0, wire_bytes = 0, raw_bytes = 0;  // this rank's share
  };
  using WindowHook = std::function<void(const std::vector<LayerSpec>& window, const DevicePlan& dp)>;
  RsCounts sharded(ShardedOp op, const std::vector<LayerSpec>& shard_layers, int dtype, bool skip_incomplete,
                   const void* in, void* out, uint64_t S, float prescale, const RngParams& rng, cudaStream_t stream,
                   int max_lanes = 0, const WindowHook& before_launch = nullptr, WireCodec codec = kMaxMin,
                   float* out_scales = nullptr);
  // builds and uploads the plans of every window without launching anything
  void prepare_sharded(const std::vector<LayerSpec>& shard_layers, int dtype, bool skip_incomplete,
                       cudaStream_t stream, int max_lanes = 0);
  // reduce_scatter_windows for this heap (cached per shard table); the all-gather uses the same
  // windows, since its per-chunk wire is the reduce-scatter's
  const std::vector<std::vector<LayerSpec>>& rs_windows(const std::vector<LayerSpec>& shard_layers, int dtype,
                                                        bool skip_incomplete, int max_lanes);

  // Compressed all-to-all (a2a_kernel), one launch whatever the splits. in_counts[q] elements of
  // `in` (consecutive, in rank order) go to rank q; out_counts[q] elements from rank q land in `out`
  // (consecutive, in rank order). My own chunk is copied; every other chunk is decode(Q(chunk)) with
  // `bits` (1..8; >= 32 moves it raw) and buckets of `bucket` counted from the chunk's first
  // element. `codec` says what the bytes of the 8-bit records mean (common/quant_math.h): max-min
  // levels, or an FP8 code per element with a per-bucket scale (bits 8, round to nearest; the caller
  // rejects stochastic rounding). The counts of a pair must agree on both ends (the caller's contract, as with NCCL).
  // Throws std::invalid_argument on a malformed call before anything is launched.
  // With a `route` that has an index, the routed kernel gathers the sent rows and scatters the
  // received ones by index; that needs a2a_rows_fit(route->row, bits, bucket, dtype) (else
  // std::invalid_argument: the caller composes index_select / index_copy_ around a plain call).
  // With `out_scales` (an FP8 codec) `out` receives the codes and out_scales the units of every chunk,
  // undecoded, the own chunk encoded by the same encoder (A2aParams::out_scales).
  // `rank_base`: the world rank of the heap's rank 0 (A2aParams::rank_base), 0 on one node.
  struct A2aCounts {
    uint64_t launches = 0, wire_bytes = 0, raw_bytes = 0;  // this rank's sends
  };
  A2aCounts all_to_all(const void* in, void* out, const std::vector<uint64_t>& in_counts,
                       const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec,
                       uint32_t bucket, const RngParams& rng, cudaStream_t stream, const A2aRoute* route = nullptr,
                       float* out_scales = nullptr, int rank_base = 0);

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
  uint64_t generation() const { return plans_.generation(); }
  uint32_t epoch() const { return epoch_; }
  size_t num_plans() const { return plans_.size(); }

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
  static constexpr size_t kMaxCachedPlans = 1024;
  PlanCache plans_{kMaxCachedPlans};  // no byte bound
  const DevicePlan* prepare_impl(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                                 cudaStream_t stream, int plan_world, uint32_t capacity, int max_lanes);
  void launch(const DevicePlan& dp, void* data, float prescale, const RngParams& rng, cudaStream_t stream,
              bool oneshot, void* out = nullptr, uint64_t out_shift = 0, bool gather = false,
              WireCodec codec = kMaxMin, float* out_scales = nullptr, uint32_t out_bucket = 0);
  std::unordered_map<uint64_t, std::vector<std::vector<LayerSpec>>> rs_windows_;
};

}  // namespace cgx

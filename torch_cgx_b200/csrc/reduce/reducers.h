// Transport-agnostic reducers: compressed Scatter-Reduce-AllGather, ring, and
// the debug all-to-all, written against Communicator + BlockBackend so the same
// code runs on host memory over Gloo (CPU tensors, tests) and on device memory
// over NCCL send/recv (cross-node stage, and the "reference-structure" baseline
// CGX_INNER_COMMUNICATOR_TYPE=NCCL).
//
// Reference: Reducer / MPI_Allreduce_ScatterReduceAllgather / MPI_Allreduce_Ring /
// NCCL_Reduce (/root/reference/src/common/reducer.{h,cc},
// scatter_reduce_allgather.cc:94-413, ring.cc:57-226, nccl_reduce.cc:89-213).
// Differences: accumulation is fp32 in rank order (bit-identical to the fused
// kernel and to the CPU oracle); quantize/dequantize run as ONE launch per
// chunk over the plan's block table instead of 2-3 launches per layer slice.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <memory>
#include <vector>

#include "../comm/communicator.h"
#include "../common/config.h"
#include "../common/plan.h"
#include "../common/sra_sim.h"
#include "block_backend.h"
#include "plan_cache.h"

namespace cgx {

class Reducer {
 public:
  Reducer(Communicator* comm, BlockBackend* ops);
  virtual ~Reducer();
  virtual const char* name() const = 0;
  // in-place allreduce of data[T] restricted to `layers`. An FP8 `codec` (layers of bits 8 or 32,
  // round to nearest) sends the compressed layers' 8-bit records as FP8 codes and adds each decoded
  // value with its own rounding; raw layers are unchanged. The debug all-to-all reduction has no FP8
  // form and throws std::invalid_argument (kAllToAllNoFp8) before anything is sent.
  virtual void allreduce(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete,
                         float prescale, const RngParams& rng, cudaStream_t stream, WireCodec codec = kMaxMin) = 0;
  // raw broadcast of `bytes` from group rank `root`
  void broadcast(void* data, size_t bytes, int root, cudaStream_t stream);
  // Compressed broadcast of `layers` (reference: Reducer::Broadcast with do_compression,
  // /root/reference/src/common/reducer.cc:96-160): the root quantizes, decodes its own bytes back
  // into `data` (so it holds exactly what every receiver will decode) and sends the SAME packed
  // bytes to every peer; receivers decode. Raw layers travel as T inside the same record. An FP8
  // `codec` as in allreduce.
  void broadcast_compressed(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete,
                            int root, const RngParams& rng, cudaStream_t stream, WireCodec codec = kMaxMin);
  // Compressed reduce-scatter over the communicator's W ranks, the scatter phase of the SRA alone.
  // `shard_layers` is ONE shard's table (offsets from the shard start, tiling [0, S)); the plan is
  // that table replicated W times at stride S, so chunk c is copy c and buckets are counted from each
  // shard's start. `in` holds W * S elements, `out` receives shard rank():
  //   out = T(prescale * in[r] + sum over peers q, in rank order, of decode(Q_q(prescale * in_q[r])))
  // accumulated in fp32 and stored once in the dtype, not requantized. Bitwise the fused rs_kernel
  // (same plan, primitives, order and RNG streams: rank q's phase-0 stream, full-buffer indices).
  // An FP8 `codec` (8-bit layers) quantizes the compressed layers with its records, round to nearest,
  // and adds each decoded value with its own rounding; raw layers are unchanged. The same for all_gather.
  void reduce_scatter(const void* in, void* out, int dtype, const std::vector<LayerSpec>& shard_layers,
                      bool skip_incomplete, float prescale, const RngParams& rng, cudaStream_t stream,
                      WireCodec codec = kMaxMin);
  // Compressed all-gather: the compressed broadcast with every rank as a root. `in` holds this rank's
  // shard of S elements, `out` W * S; rank q quantizes its shard once (copy q of the replicated table,
  // its phase-1 stream), decodes it into its own chunk and sends the same bytes to every peer, which
  // decode them. Every rank's `out` is the same bytes, bitwise the fused ag_kernel's; raw layers
  // (bits 32) are copied unchanged. `in` may be `out`'s chunk rank(), or disjoint from it.
  // With `out_scales` (the codes output, check_sharded_buffers) every chunk's records are unpacked
  // instead of decoded (BlockBackend::unpack_fp8) into the codes `out` and the units out_scales, the
  // own one from the record this rank sends: bitwise the fused ag_kernel's codes output, with the
  // decoded call's wire.
  void all_gather(const void* in, void* out, int dtype, const std::vector<LayerSpec>& shard_layers,
                  bool skip_incomplete, const RngParams& rng, cudaStream_t stream, WireCodec codec = kMaxMin,
                  float* out_scales = nullptr);
  // Compressed all-to-all over the communicator's W ranks, bitwise FusedSra::all_to_all (same
  // arguments and checks): each chunk for a peer is quantized by the standalone item kernels through
  // a one-layer plan of the chunk, the records are exchanged and every peer's chunk is decoded into
  // its rows; the own chunk is copied, and with bits >= 32 every chunk travels as its bytes. An FP8
  // `codec` quantizes and decodes the 8-bit records with the block backend's FP8 primitives. With
  // `out_scales` (an FP8 codec) the records are unpacked instead of decoded (BlockBackend::unpack_fp8)
  // into the codes `out` and the units out_scales, and the own chunk is quantized into a record and
  // unpacked too: bitwise the fused kernel's codes output. `rank_base` is the world rank of the
  // communicator's rank 0: the chunk from rank q to rank p uses a2a_rng_stream(rank_base + q,
  // rank_base + p), the stream it has in an all-to-all of all the world's ranks.
  void all_to_all(const void* in, void* out, const std::vector<uint64_t>& in_counts,
                  const std::vector<uint64_t>& out_counts, int dtype, int bits, WireCodec codec, uint32_t bucket,
                  const RngParams& rng, cudaStream_t stream, float* out_scales = nullptr, int rank_base = 0);
  uint64_t bytes_sent() const { return bytes_sent_; }
  size_t num_plans() const { return plans_.size(); }
  uint64_t plan_uploads() const { return plans_.uploads(); }

 protected:
  // The plan of `layers`, uploaded when the backend is the device's. world <= 0: one chunk per rank
  // of the communicator; otherwise that many chunks. A call never uses a plan after it has asked for
  // another: the request may drop the cache, which frees every earlier plan (after synchronising
  // `stream`, so no kernel still reads them).
  const DevicePlan& plan_for(const std::vector<LayerSpec>& layers, int dtype, bool skip_incomplete,
                             cudaStream_t stream, int world = 0);
  uint8_t* scratch(int slot, size_t bytes);  // grow-only scratch buffers of the backend's memory kind
  void all_to_all_codes(const void* in, uint8_t* codes, float* scales, const std::vector<uint64_t>& in_counts,
                        const std::vector<uint64_t>& out_counts, int dtype, WireCodec codec, uint32_t bucket,
                        const RngParams& rng, cudaStream_t stream, int rank_base);
  static size_t row_bytes(const Plan& p) { return ((size_t)p.max_chunk_wire + 255) / 256 * 256; }
  // [first element, one past last element) spanned by the blocks of a chunk / of the whole plan
  static void chunk_span(const Plan& p, int chunk, uint32_t* lo, uint32_t* hi);

  Communicator* comm_;
  BlockBackend* ops_;
  uint64_t bytes_sent_ = 0;

 private:
  // Bounded, since tensor sizes and MoE splits may change every call. Both figures are design
  // choices, not measurements: 256 plans covers the layouts of a training step with room to spare,
  // and 64 MiB of tables is about four million warp items, the tables of some 2G elements.
  static constexpr size_t kMaxPlans = 256;
  static constexpr size_t kMaxTableBytes = 64ull << 20;
  PlanCache plans_{kMaxPlans, kMaxTableBytes};
  struct Buf {
    uint8_t* p = nullptr;
    size_t cap = 0;
  };
  std::vector<Buf> bufs_;
};

class SraReducer : public Reducer {
 public:
  using Reducer::Reducer;
  const char* name() const override { return "SRA"; }
  void allreduce(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete, float prescale,
                 const RngParams& rng, cudaStream_t stream, WireCodec codec) override;
};

class RingReducer : public Reducer {
 public:
  using Reducer::Reducer;
  const char* name() const override { return "RING"; }
  void allreduce(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete, float prescale,
                 const RngParams& rng, cudaStream_t stream, WireCodec codec) override;
};

// Debug variant (CGX_DEBUG_ALL_TO_ALL_REDUCTION): every rank quantizes the whole
// buffer once, sends it to everybody and adds everything it receives to its own
// raw values -- one quantization error per peer, replicas NOT bit-identical.
class AllToAllReducer : public Reducer {
 public:
  using Reducer::Reducer;
  const char* name() const override { return "ALLTOALL"; }
  void allreduce(void* data, int dtype, const std::vector<LayerSpec>& layers, bool skip_incomplete, float prescale,
                 const RngParams& rng, cudaStream_t stream, WireCodec codec) override;
};

constexpr const char* kAllToAllNoFp8 =
    "cgx: the debug all-to-all reduction (CGX_DEBUG_ALL_TO_ALL_REDUCTION) has no FP8 formats";

std::unique_ptr<Reducer> make_reducer(ReductionType type, Communicator* comm, BlockBackend* ops);

}  // namespace cgx

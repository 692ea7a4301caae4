// torch.distributed backend "cgx".
//
// Capabilities mirror ProcessGroupCGX of the reference
// (/root/reference/src/ProcessGroupCGX.h:105-317, .cc:269-833): allreduce of
// CUDA fp16/fp32 (+bf16 here) SUM tensors goes through the compressed
// allreduce engine on a dedicated side stream; everything else is forwarded
// verbatim -- there to MPI, here to an internal Gloo (CPU tensors) or NCCL
// (CUDA tensors) delegate, which also supplies the collectives the reference
// throws on (reduce_scatter, _allgather_base, allreduce_coalesced).
//
// Architecture differences (H100-first):
//  * no worker thread / FIFO queue on the CUDA path (reference .cc:300-339): the
//    whole allreduce is ONE stream-ordered kernel launch, so the Work/Future is
//    completed at enqueue time with CUDA events, like ProcessGroupNCCL;
//  * the start event is recorded on the CALLER's current stream (the reference
//    records on the worker thread's default stream -- SURVEY.md §2.8 #8) and
//    every Work owns its end event;
//  * rendezvous uses the c10d Store handed to the constructor (the reference
//    ignores store/timeout and requires mpirun -- .cc:259-267).
#pragma once
#include <ATen/cuda/CUDAEvent.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/csrc/distributed/c10d/Backend.hpp>
#include <torch/csrc/distributed/c10d/Store.hpp>
#include <torch/csrc/distributed/c10d/Work.hpp>

#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <optional>
#include <string>
#include <vector>

#include "../engine/engine.h"

namespace cgx {

class ProcessGroupCGX;

// Work of one engine allreduce. Like ProcessGroupNCCL it is "complete" for stream-ordering purposes
// as soon as the kernel is enqueued (wait() makes the caller's stream wait on the end event, the
// CUDA-aware Future carries the same event). Failures are asynchronous: when a fused kernel
// reports a timeout / abort in the host-mapped status word, the backend's watchdog stores the
// error in every Work still in flight (isSuccess() / exception() / wait() then report it) and
// every later collective fails fast. With CGX_BLOCKING_WAIT=1, wait() blocks the host until the
// kernel has finished and throws right there.
// Reference: WorkMPI + finishWorkMPIError (/root/reference/src/ProcessGroupCGX.cc:120-142, :312-317).
class WorkCGX : public c10d::Work {
 public:
  WorkCGX(int rank, c10d::OpType op, const char* title, std::vector<at::Tensor> outputs, c10::Device device,
          c10::cuda::CUDAStream comm_stream, ProcessGroupCGX* owner);
  bool isCompleted() override;
  bool wait(std::chrono::milliseconds timeout = kNoTimeout) override;
  void synchronize() override;
  std::vector<at::Tensor> result() override;
  c10::intrusive_ptr<c10::ivalue::Future> getFuture() override;
  // record the end of the work on the comm stream and complete the future
  void finish_on_stream();
  // the collective was refused (group already failed / aborted): Work and Future carry the error
  void fail_now(std::exception_ptr e);
  // the watchdog found a device-side failure while this Work was in flight
  void set_error(std::exception_ptr e);
  bool gpu_done() const { return end_recorded_ && end_event_.query(); }

 private:
  std::vector<at::Tensor> outputs_;
  c10::Device device_;
  c10::cuda::CUDAStream comm_stream_;
  at::cuda::CUDAEvent end_event_;
  at::cuda::CUDAEvent start_event_;  // per Work: nothing shared between calls (SURVEY.md §2.8 #8)
  bool end_recorded_ = false;
  ProcessGroupCGX* owner_;
  c10::intrusive_ptr<c10::ivalue::Future> future_;
  friend class ProcessGroupCGX;
};

// Delegates of the node-local and cross-node sub-groups (hierarchical allreduce);
// all optional. `local_size` consecutive ranks form a node.
struct CgxTopology {
  int local_size = 0;  // 0 = whole group is one node
  c10::intrusive_ptr<c10d::Backend> cpu_local, cpu_cross, cuda_local, cuda_cross;
};

// Host-side worker: a single thread draining a FIFO of jobs, the role of
// ProcessGroupCGX::runLoop / enqueue in the reference (/root/reference/src/
// ProcessGroupCGX.cc:300-339). Only the *host-tensor* compressed allreduce uses it
// (blocking Gloo send/recv must not stall the autograd thread); the CUDA path
// needs no thread because it is a single stream-ordered kernel launch.
class HostWorker {
 public:
  HostWorker();
  ~HostWorker();
  void submit(std::function<void()> job);
  void drain();  // block until every submitted job has finished

 private:
  void loop();
  std::mutex mu_;
  std::condition_variable cv_, idle_cv_;
  std::deque<std::function<void()>> q_;
  bool stop_ = false;
  bool busy_ = false;
  std::thread th_;
};

class ProcessGroupCGX : public c10d::Backend {
 public:
  using Topology = CgxTopology;

  ProcessGroupCGX(const c10::intrusive_ptr<c10d::Store>& store, int rank, int size,
                  std::chrono::milliseconds timeout, c10::intrusive_ptr<c10d::Backend> cpu_delegate,
                  c10::intrusive_ptr<c10d::Backend> cuda_delegate, Topology topo = Topology());
  ~ProcessGroupCGX() override;

  const std::string getBackendName() const override { return "cgx"; }

  c10::intrusive_ptr<c10d::Work> allreduce(std::vector<at::Tensor>& tensors,
                                           const c10d::AllreduceOptions& opts = c10d::AllreduceOptions()) override;
  c10::intrusive_ptr<c10d::Work> allreduce_coalesced(
      std::vector<at::Tensor>& tensors,
      const c10d::AllreduceCoalescedOptions& opts = c10d::AllreduceCoalescedOptions()) override;
  c10::intrusive_ptr<c10d::Work> broadcast(std::vector<at::Tensor>& tensors,
                                           const c10d::BroadcastOptions& opts = c10d::BroadcastOptions()) override;
  c10::intrusive_ptr<c10d::Work> reduce(std::vector<at::Tensor>& tensors,
                                        const c10d::ReduceOptions& opts = c10d::ReduceOptions()) override;
  c10::intrusive_ptr<c10d::Work> allgather(std::vector<std::vector<at::Tensor>>& outputTensors,
                                           std::vector<at::Tensor>& inputTensors,
                                           const c10d::AllgatherOptions& opts = c10d::AllgatherOptions()) override;
  c10::intrusive_ptr<c10d::Work> _allgather_base(at::Tensor& outputBuffer, at::Tensor& inputBuffer,
                                                 const c10d::AllgatherOptions& opts = c10d::AllgatherOptions()) override;
  c10::intrusive_ptr<c10d::Work> allgather_coalesced(std::vector<std::vector<at::Tensor>>& outputTensorLists,
                                                     std::vector<at::Tensor>& inputTensors,
                                                     const c10d::AllgatherOptions& opts = c10d::AllgatherOptions()) override;
  c10::intrusive_ptr<c10d::Work> allgather_into_tensor_coalesced(
      std::vector<at::Tensor>& outputs, std::vector<at::Tensor>& inputs,
      const c10d::AllgatherOptions& opts = c10d::AllgatherOptions()) override;
  c10::intrusive_ptr<c10d::Work> gather(std::vector<std::vector<at::Tensor>>& outputTensors,
                                        std::vector<at::Tensor>& inputTensors,
                                        const c10d::GatherOptions& opts = c10d::GatherOptions()) override;
  c10::intrusive_ptr<c10d::Work> scatter(std::vector<at::Tensor>& outputTensors,
                                         std::vector<std::vector<at::Tensor>>& inputTensors,
                                         const c10d::ScatterOptions& opts = c10d::ScatterOptions()) override;
  c10::intrusive_ptr<c10d::Work> reduce_scatter(std::vector<at::Tensor>& outputTensors,
                                                std::vector<std::vector<at::Tensor>>& inputTensors,
                                                const c10d::ReduceScatterOptions& opts = c10d::ReduceScatterOptions()) override;
  c10::intrusive_ptr<c10d::Work> _reduce_scatter_base(at::Tensor& outputBuffer, at::Tensor& inputBuffer,
                                                      const c10d::ReduceScatterOptions& opts = c10d::ReduceScatterOptions()) override;
  c10::intrusive_ptr<c10d::Work> reduce_scatter_tensor_coalesced(
      std::vector<at::Tensor>& outputs, std::vector<at::Tensor>& inputs,
      const c10d::ReduceScatterOptions& opts = c10d::ReduceScatterOptions()) override;
  c10::intrusive_ptr<c10d::Work> alltoall_base(at::Tensor& outputBuffer, at::Tensor& inputBuffer,
                                               std::vector<int64_t>& outputSplitSizes,
                                               std::vector<int64_t>& inputSplitSizes,
                                               const c10d::AllToAllOptions& opts = c10d::AllToAllOptions()) override;
  c10::intrusive_ptr<c10d::Work> alltoall(std::vector<at::Tensor>& outputTensors,
                                          std::vector<at::Tensor>& inputTensors,
                                          const c10d::AllToAllOptions& opts = c10d::AllToAllOptions()) override;
  c10::intrusive_ptr<c10d::Work> send(std::vector<at::Tensor>& tensors, int dstRank, int tag) override;
  c10::intrusive_ptr<c10d::Work> recv(std::vector<at::Tensor>& tensors, int srcRank, int tag) override;
  c10::intrusive_ptr<c10d::Work> recvAnysource(std::vector<at::Tensor>& tensors, int tag) override;
  c10::intrusive_ptr<c10d::Work> barrier(const c10d::BarrierOptions& opts = c10d::BarrierOptions()) override;

  void setSequenceNumberForGroup() override {}
  uint64_t getSequenceNumberForGroup() override { return seq_; }

  // Make every spinning kernel of this group give up, fail everything in flight and refuse new
  // collectives (reference: ProcessGroupCGX::abort -> MPI_Abort, ProcessGroupCGX.cc:295-298; here
  // the process survives and sees RuntimeErrors).
  void abort() override;
  void shutdown() override;

  // ---- cgx-specific API (bound to Python) ----------------------------------
  // allreduce of one DDP bucket whose index is known (no cursor guessing);
  // average == true fuses the 1/world scale into the kernel.
  c10::intrusive_ptr<c10d::Work> allreduce_bucket(at::Tensor& tensor, int64_t bucket_idx, bool average);
  // Compressed reduce-scatter or all-gather through the fused P2P kernel; the c10d entry points of
  // both stay with the delegate.
  //  kReduceScatter (reduce_scatter_tensor semantics): `in` holds size() * out.numel() elements,
  //  rank r receives shard r.
  //  kAllGather (all_gather_into_tensor semantics): `out` holds size() * in.numel() elements,
  //  chunk q is rank q's shard. Every shard, this rank's own included, arrives as one quantization
  //  round trip, so every rank's `out` is the same. average and skip_incomplete are false.
  // The shard may be this rank's chunk of the full buffer. `layers`: quantization table of one
  // shard, (elem_off, numel, bits, bucket) relative to the shard start, empty = one layer with
  // `bits` / `bucket_size`. seed < 0: CGX_SEED. overlapped: at most CGX_OVERLAP_LANES CTAs (runs
  // beside compute).
  c10::intrusive_ptr<c10d::Work> sharded_compressed(ShardedOp op, at::Tensor& out, at::Tensor& in, bool average,
                                                    int bits, int bucket_size, bool skip_incomplete, bool stochastic,
                                                    int64_t seed, bool overlapped,
                                                    const std::vector<LayerSpec>& layers);
  // force the lazy CUDA-side initialisation (heap allocation + IPC exchange)
  void init_cuda(int64_t device_index);
  bool p2p_ready() const { return engine_ && engine_->has_p2p(); }
  int64_t local_size() const { return engine_ ? engine_->local_size() : getSize(); }
  int64_t lanes() const;
  std::vector<int64_t> stats() const;  // calls, kernel launches, elements, wire bytes, raw bytes
  void reset_stats();
  void check_health();
  // empty when healthy, else the first failure this group has seen
  std::string failure() const;
  bool blocking_wait() const { return blocking_wait_; }
  int64_t last_lanes() const { return engine_ && engine_->has_p2p() ? engine_->fused()->last_lanes() : 0; }
  bool uses_multicast() const { return engine_ && engine_->has_p2p() && engine_->fused()->uses_multicast(); }
  std::string heap_kind() const {
    if (!engine_ || !engine_->heap()) return "none";
    return engine_->heap()->kind() == HeapKind::kVmm ? "vmm" : "cudaMalloc";
  }
  // per-lane device timestamps of the last fused allreduce (see FusedSra::read_trace)
  void enable_trace(bool on);
  at::Tensor read_trace();

 private:
  c10::intrusive_ptr<c10d::Backend> delegate_for(const at::Tensor& t, const char* op);
  bool eligible_for_engine(const at::Tensor& t, const c10d::ReduceOp& op) const;
  // The Work of one collective on the comm stream: refused once the group has failed; otherwise,
  // under mu_, ordered after the caller's stream, `in` (may be null) and `out` recorded on the comm
  // stream, run(comm stream) enqueues the engine call; then registered with the watchdog.
  template <class Run>
  c10::intrusive_ptr<c10d::Work> enqueue_cuda(c10d::OpType op, const char* title, at::Tensor& out,
                                              const at::Tensor* in, Run&& run);
  c10::intrusive_ptr<c10d::Work> engine_allreduce(at::Tensor& t, bool average, int bucket_idx);
  c10::intrusive_ptr<c10d::Work> engine_allreduce_cpu(at::Tensor& t, bool average, int bucket_idx);
  void ensure_cuda(c10::DeviceIndex dev);

  c10::intrusive_ptr<c10d::Store> store_;
  std::chrono::milliseconds timeout_;
  c10::intrusive_ptr<c10d::Backend> cpu_delegate_;
  c10::intrusive_ptr<c10d::Backend> cuda_delegate_;
  Topology topo_;
  bool compress_cpu_ = false;  // CGX_COMPRESS_CPU: route CPU float tensors through the generic reducers
  bool cuda_ready_ = false;
  EngineConfig cfg_;
  std::unique_ptr<AllreduceEngine> engine_;
  std::optional<c10::cuda::CUDAStream> comm_stream_;
  c10::DeviceIndex device_ = -1;
  std::mutex mu_;
  uint64_t seq_ = 0;
  std::unique_ptr<HostWorker> worker_;  // created on first use

  // ---- failure detection -------------------------------------------------------------------
  // returns the failure (recording it on first sight) or an empty string
  std::string poll_failure();
  void fail_inflight(const std::string& msg);
  void watchdog_loop();
  bool blocking_wait_ = false;
  mutable std::mutex fail_mu_;
  std::string failure_;                 // first failure seen (sticky)
  std::deque<c10::weak_intrusive_ptr<WorkCGX>> inflight_;
  std::thread watchdog_;
  std::condition_variable watchdog_cv_;
  bool watchdog_stop_ = false;
  friend class WorkCGX;
};

}  // namespace cgx

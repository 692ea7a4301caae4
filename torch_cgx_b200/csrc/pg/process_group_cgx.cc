#include "process_group_cgx.h"

#include <c10/cuda/CUDACachingAllocator.h>
#include <c10/cuda/CUDAGraphsC10Utils.h>
#include <c10/cuda/CUDAGuard.h>

#include <algorithm>
#include <cstring>

#include "../kernels/launch.h"
#include "c10d_communicator.h"

namespace cgx {

namespace {

int to_cgx_dtype(at::ScalarType t) {
  switch (t) {
    case at::kFloat: return kF32;
    case at::kHalf: return kF16;
    case at::kBFloat16: return kBF16;
    default: return -1;
  }
}

// KVStore over the c10d Store handed to the backend
class C10dKV : public KVStore {
 public:
  explicit C10dKV(c10::intrusive_ptr<c10d::Store> s) : s_(std::move(s)) {}
  void set(const std::string& key, const std::vector<uint8_t>& value) override { s_->set(key, value); }
  std::vector<uint8_t> get(const std::string& key) override { return s_->get(key); }

 private:
  c10::intrusive_ptr<c10d::Store> s_;
};

}  // namespace

// ---------------------------------------------------------------- WorkCGX ---
WorkCGX::WorkCGX(int rank, c10d::OpType op, const char* title, std::vector<at::Tensor> outputs,
                 c10::Device device, c10::cuda::CUDAStream comm_stream, ProcessGroupCGX* owner)
    : c10d::Work(rank, op, title, std::optional<std::vector<at::Tensor>>(outputs)),
      outputs_(std::move(outputs)),
      device_(device),
      comm_stream_(comm_stream),
      end_event_(cudaEventDisableTiming),
      start_event_(cudaEventDisableTiming),
      owner_(owner) {
  future_ = c10::make_intrusive<c10::ivalue::Future>(c10::ListType::create(c10::TensorType::get()),
                                                     std::vector<c10::Device>{device_});
}

void WorkCGX::finish_on_stream() {
  end_event_.record(comm_stream_);
  end_recorded_ = true;
  {
    // the Future records its own events on the *current* stream of its devices:
    // make that the comm stream so .then() callbacks / wait() order after the kernel
    c10::cuda::CUDAStreamGuard g(comm_stream_);
    future_->markCompleted(at::IValue(outputs_));
  }
  finish();  // completed_ = true (the GPU work itself is tracked by end_event_)
}

void WorkCGX::fail_now(std::exception_ptr e) {
  future_->setError(e);
  finish(e);
}

void WorkCGX::set_error(std::exception_ptr e) {
  std::lock_guard<std::mutex> g(mutex_);
  if (!exception_) exception_ = e;
}

bool WorkCGX::isCompleted() { return !end_recorded_ || end_event_.query(); }

void WorkCGX::synchronize() {
  if (end_recorded_) end_event_.block(c10::cuda::getCurrentCUDAStream(device_.index()));
}

bool WorkCGX::wait(std::chrono::milliseconds /*timeout*/) {
  // CUDA semantics of c10d: make the caller's current stream wait, never block the host ...
  synchronize();
  // ... unless asked to (CGX_BLOCKING_WAIT=1): then a device-side failure surfaces right here
  if (end_recorded_ && owner_ != nullptr && owner_->blocking_wait()) {
    end_event_.synchronize();
    const std::string msg = owner_->poll_failure();
    if (!msg.empty()) set_error(std::make_exception_ptr(std::runtime_error(msg)));
  }
  std::exception_ptr e;
  {
    std::lock_guard<std::mutex> g(mutex_);
    e = exception_;
  }
  if (e) std::rethrow_exception(e);
  return true;
}
std::vector<at::Tensor> WorkCGX::result() { return outputs_; }
c10::intrusive_ptr<c10::ivalue::Future> WorkCGX::getFuture() { return future_; }

// ------------------------------------------------------------- HostWorker ---
HostWorker::HostWorker() : th_([this] { loop(); }) {}

HostWorker::~HostWorker() {
  {
    std::lock_guard<std::mutex> g(mu_);
    stop_ = true;
  }
  cv_.notify_all();
  if (th_.joinable()) th_.join();
}

void HostWorker::submit(std::function<void()> job) {
  {
    std::lock_guard<std::mutex> g(mu_);
    q_.push_back(std::move(job));
  }
  cv_.notify_one();
}

void HostWorker::drain() {
  std::unique_lock<std::mutex> g(mu_);
  idle_cv_.wait(g, [this] { return q_.empty() && !busy_; });
}

void HostWorker::loop() {
  for (;;) {
    std::function<void()> job;
    {
      std::unique_lock<std::mutex> g(mu_);
      cv_.wait(g, [this] { return stop_ || !q_.empty(); });
      if (q_.empty()) return;  // stop requested and nothing left
      job = std::move(q_.front());
      q_.pop_front();
      busy_ = true;
    }
    job();  // jobs report their own errors through their futures
    {
      std::lock_guard<std::mutex> g(mu_);
      busy_ = false;
    }
    idle_cv_.notify_all();
  }
}

// -------------------------------------------------------- ProcessGroupCGX ---
ProcessGroupCGX::ProcessGroupCGX(const c10::intrusive_ptr<c10d::Store>& store, int rank, int size,
                                 std::chrono::milliseconds timeout,
                                 c10::intrusive_ptr<c10d::Backend> cpu_delegate,
                                 c10::intrusive_ptr<c10d::Backend> cuda_delegate, Topology topo)
    : c10d::Backend(rank, size),
      store_(store),
      timeout_(timeout),
      cpu_delegate_(std::move(cpu_delegate)),
      cuda_delegate_(std::move(cuda_delegate)),
      topo_(std::move(topo)),
      cfg_(EngineConfig::read()) {
  compress_cpu_ = env_bool("CGX_COMPRESS_CPU", false);
  blocking_wait_ = env_bool("CGX_BLOCKING_WAIT", false);
  engine_ = std::make_unique<AllreduceEngine>(rank, size, cfg_);
  engine_->set_topology(topo_.local_size > 0 ? topo_.local_size : size);
  TORCH_CHECK(engine_->local_size() <= kMaxPeers || cfg_.inner_comm != CommType::kP2P,
              "cgx: the P2P path supports at most ", kMaxPeers, " ranks per node");
  // host-memory reducers (Gloo transport): whole group when single-node, else local + cross sub-groups
  {
    std::unique_ptr<Communicator> intra, cross;
    if (engine_->nodes() > 1) {
      if (topo_.cpu_local && engine_->local_size() > 1)
        intra = std::make_unique<C10dCommunicator>(topo_.cpu_local, false, -1);
      if (topo_.cpu_cross) cross = std::make_unique<C10dCommunicator>(topo_.cpu_cross, false, -1);
    } else if (cpu_delegate_ && size > 1) {
      intra = std::make_unique<C10dCommunicator>(cpu_delegate_, false, -1);
    }
    if (intra || cross || size == 1) engine_->attach_generic(false, std::move(intra), std::move(cross));
  }
  log_msg(1, "cgx[%d/%d]: backend created (inner=%s/%s fusion=%lld MB lanes=%d)", rank, size,
          to_string(cfg_.inner_comm), to_string(cfg_.inner_reduction), (long long)(cfg_.fusion_bytes >> 20),
          cfg_.lanes);
}

ProcessGroupCGX::~ProcessGroupCGX() {
  {
    std::lock_guard<std::mutex> g(fail_mu_);
    watchdog_stop_ = true;
  }
  watchdog_cv_.notify_all();
  if (watchdog_.joinable()) watchdog_.join();
  worker_.reset();  // finishes queued host jobs before the engine goes away
  if (engine_ && device_ >= 0) {
    c10::cuda::CUDAGuard g(device_);
    cudaDeviceSynchronize();
  }
  engine_.reset();
}

c10::intrusive_ptr<c10d::Backend> ProcessGroupCGX::delegate_for(const at::Tensor& t, const char* op) {
  if (t.is_cuda()) {
    TORCH_CHECK(cuda_delegate_, "cgx: no CUDA delegate backend available for ", op);
    return cuda_delegate_;
  }
  TORCH_CHECK(cpu_delegate_, "cgx: no CPU delegate backend available for ", op);
  return cpu_delegate_;
}

bool ProcessGroupCGX::eligible_for_engine(const at::Tensor& t, const c10d::ReduceOp& op) const {
  // reference: do_compress = (fp16|fp32) && SUM && CUDA  (ProcessGroupCGX.cc:374-377); bf16 and AVG added
  if (to_cgx_dtype(t.scalar_type()) < 0) return false;
  if (!(op == c10d::ReduceOp::SUM || op == c10d::ReduceOp::AVG)) return false;
  if (!t.is_non_overlapping_and_dense()) return false;
  if (!t.is_cuda()) return compress_cpu_ && engine_->has_generic(false);
  if (cfg_.inner_comm == CommType::kP2P) return true;
  // NCCL transport (reference-structure path): needs a CUDA delegate to carry the bytes
  return cuda_delegate_ != nullptr || getSize() == 1;
}

void ProcessGroupCGX::init_cuda(int64_t device_index) { ensure_cuda((c10::DeviceIndex)device_index); }

void ProcessGroupCGX::ensure_cuda(c10::DeviceIndex dev) {
  std::lock_guard<std::mutex> lk(mu_);
  if (cuda_ready_) {
    TORCH_CHECK(dev == device_, "cgx: this process group is bound to cuda:", (int)device_,
                " but got a tensor on cuda:", (int)dev);
    return;
  }
  c10::cuda::CUDAGuard g(dev);
  device_ = dev;
  comm_stream_ = c10::cuda::getStreamFromPool(/*isHighPriority=*/true, dev);
  const int lsize = engine_->local_size(), lrank = engine_->local_rank(), node = engine_->node();

  // device-memory generic reducers (NCCL send/recv transport): cross-node stage, intra-node
  // broadcast in leader mode, and the whole intra-node stage when CGX_INNER_COMMUNICATOR_TYPE=NCCL
  {
    std::unique_ptr<Communicator> intra, cross;
    if (engine_->nodes() > 1) {
      if (topo_.cuda_local && lsize > 1) intra = std::make_unique<C10dCommunicator>(topo_.cuda_local, true, dev);
      if (topo_.cuda_cross) cross = std::make_unique<C10dCommunicator>(topo_.cuda_cross, true, dev);
    } else if (cuda_delegate_ && getSize() > 1) {
      intra = std::make_unique<C10dCommunicator>(cuda_delegate_, true, dev);
    }
    engine_->attach_generic(true, std::move(intra), std::move(cross));
  }

  if (cfg_.inner_comm == CommType::kP2P) {
    // agree on the number of lanes (CTAs): min over the node's ranks of what can be co-resident
    int resident = sra_max_resident_ctas(kF32);
    int want = cfg_.lanes > 0 ? cfg_.lanes : resident;
    int mine = std::max(1, std::min(want, resident));
    C10dKV kv(store_);
    const std::string prefix = "cgx/p2p/node" + std::to_string(node);
    {
      std::vector<uint8_t> v(sizeof(int));
      std::memcpy(v.data(), &mine, sizeof(int));
      kv.set(prefix + "/lanes/" + std::to_string(lrank), v);
    }
    int lanes = mine;
    for (int p = 0; p < lsize; ++p) {
      if (p == lrank) continue;
      auto v = kv.get(prefix + "/lanes/" + std::to_string(p));
      int other = 0;
      std::memcpy(&other, v.data(), sizeof(int));
      lanes = std::min(lanes, other);
    }
    HeapLayout layout = HeapLayout::make(lsize, lanes, AllreduceEngine::required_slot_bytes(cfg_, lsize),
                                          AllreduceEngine::required_oneshot_slot_bytes(cfg_));
    auto heap = std::make_unique<SymmetricHeap>(lrank, lsize, layout);
    if (lsize > 1) heap->connect_ipc(kv, prefix);
    engine_->attach_heap(std::move(heap), lanes);
    log_msg(1, "cgx[%d]: P2P engine ready on cuda:%d (node %d, local %d/%d, lanes=%d, heap=%.1f MB, slot=%u B)",
            getRank(), (int)dev, node, lrank, lsize, lanes, (double)layout.total / (1 << 20), layout.slot_bytes);
  }
  cuda_ready_ = true;
  if (engine_->has_p2p() && !watchdog_.joinable()) watchdog_ = std::thread([this] { watchdog_loop(); });
}

// ------------------------------------------------------------ failure detection ---
std::string ProcessGroupCGX::failure() const {
  std::lock_guard<std::mutex> g(fail_mu_);
  return failure_;
}

std::string ProcessGroupCGX::poll_failure() {
  {
    std::lock_guard<std::mutex> g(fail_mu_);
    if (!failure_.empty()) return failure_;
  }
  if (!engine_ || !engine_->has_p2p()) return std::string();
  const std::string msg = engine_->fused()->status_message();  // reads host-mapped memory only
  if (msg.empty()) return msg;
  fail_inflight(msg);
  return failure();
}

void ProcessGroupCGX::fail_inflight(const std::string& msg) {
  std::deque<c10::weak_intrusive_ptr<WorkCGX>> works;
  {
    std::lock_guard<std::mutex> g(fail_mu_);
    if (!failure_.empty()) return;
    failure_ = msg;
    works.swap(inflight_);
  }
  log_msg(0, "cgx[%d]: %s", getRank(), msg.c_str());
  const std::exception_ptr e = std::make_exception_ptr(std::runtime_error(msg));
  for (auto& w : works)
    if (auto sp = w.lock()) sp->set_error(e);
}

void ProcessGroupCGX::watchdog_loop() {
  std::unique_lock<std::mutex> lk(fail_mu_);
  while (!watchdog_stop_) {
    watchdog_cv_.wait_for(lk, std::chrono::milliseconds(50));
    if (watchdog_stop_) break;
    if (!failure_.empty()) {
      inflight_.clear();  // late arrivals are failed at enqueue time
      continue;
    }
    // Works whose kernel has finished may only be forgotten once the status word has been seen
    // clean AFTER they finished: a kernel that gave up writes the status before it exits, so
    // "done, then clean" proves a clean run, while "clean, then done" would not.
    size_t done = 0;
    for (const auto& w : inflight_) {
      auto sp = w.lock();
      if (sp && !sp->gpu_done()) break;
      ++done;
    }
    lk.unlock();
    const std::string msg = poll_failure();  // on failure: marks every in-flight work, finished ones included
    lk.lock();
    if (msg.empty())
      for (; done > 0 && !inflight_.empty(); --done) inflight_.pop_front();
  }
}

void ProcessGroupCGX::abort() {
  if (engine_ && engine_->heap()) engine_->heap()->request_abort(true);
  fail_inflight("cgx: process group aborted on rank " + std::to_string(getRank()));
  if (cuda_delegate_) cuda_delegate_->abort();
  if (cpu_delegate_) cpu_delegate_->abort();
}

void ProcessGroupCGX::shutdown() {
  if (worker_) worker_->drain();
  if (cuda_delegate_) cuda_delegate_->shutdown();
  if (cpu_delegate_) cpu_delegate_->shutdown();
}

template <class Run>
c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::enqueue_cuda(c10d::OpType op, const char* title, at::Tensor& out,
                                                             const at::Tensor* in, Run&& run) {
  const c10::DeviceIndex dev = out.device().index();
  ensure_cuda(dev);
  c10::cuda::CUDAGuard g(dev);
  auto cur = c10::cuda::getCurrentCUDAStream(dev);
  auto work = c10::make_intrusive<WorkCGX>(getRank(), op, title, std::vector<at::Tensor>{out}, out.device(),
                                           *comm_stream_, this);
  {
    // a group that has failed (device timeout, abort) refuses new work: the error travels in the
    // Work and in its Future (DDP raises it from backward) instead of hanging on dead peers
    const std::string failed = poll_failure();
    if (!failed.empty()) {
      work->fail_now(std::make_exception_ptr(std::runtime_error(failed)));
      return work;
    }
  }
  {
    std::lock_guard<std::mutex> lk(mu_);
    ++seq_;
    // order after the producer of the tensors on the caller's stream
    work->start_event_.record(cur);
    work->start_event_.block(*comm_stream_);
    // the caching allocator must not hand this memory out while the comm stream uses it
    if (in != nullptr) c10::cuda::CUDACachingAllocator::recordStream(in->storage().data_ptr(), *comm_stream_);
    c10::cuda::CUDACachingAllocator::recordStream(out.storage().data_ptr(), *comm_stream_);
    run(comm_stream_->stream());
    work->finish_on_stream();
  }
  // (works created while a CUDA graph is being captured are not watched: their events belong to
  // the graph and must not be queried)
  if (engine_->has_p2p() && c10::cuda::currentStreamCaptureStatusMayInitCtx() == c10::cuda::CaptureStatus::None) {
    std::lock_guard<std::mutex> g2(fail_mu_);
    inflight_.emplace_back(work);
    if (inflight_.size() > 4096) inflight_.pop_front();
  }
  return work;
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::engine_allreduce(at::Tensor& t, bool average, int bucket_idx) {
  return enqueue_cuda(c10d::OpType::ALLREDUCE, "cgx:all_reduce", t, nullptr, [&](cudaStream_t s) {
    engine_->allreduce_cuda(t.data_ptr(), to_cgx_dtype(t.scalar_type()), t.numel(), average, bucket_idx, s,
                            /*overlapped=*/bucket_idx >= 0);
  });
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::sharded_compressed(ShardedOp op, at::Tensor& out, at::Tensor& in,
                                                                   bool average, int bits, int bucket_size,
                                                                   bool skip_incomplete, bool stochastic,
                                                                   int64_t seed, bool overlapped,
                                                                   const std::vector<LayerSpec>& layers) {
  const bool rs = op == ShardedOp::kReduceScatter;
  const char* name = op_name(op);
  TORCH_CHECK(in.is_cuda() && out.is_cuda(), "cgx: ", name, "_compressed needs CUDA tensors");
  TORCH_CHECK(in.device() == out.device(), "cgx: ", name, "_compressed: input and output on different devices");
  const int dtype = to_cgx_dtype(in.scalar_type());
  TORCH_CHECK(dtype >= 0 && out.scalar_type() == in.scalar_type(), "cgx: ", name,
              "_compressed needs float32, float16 or bfloat16 tensors of one dtype, got ", in.scalar_type(), " and ",
              out.scalar_type());
  TORCH_CHECK(in.is_contiguous() && out.is_contiguous(), "cgx: ", name, "_compressed needs contiguous tensors");
  const at::Tensor& full = rs ? in : out;
  const at::Tensor& shard = rs ? out : in;
  TORCH_CHECK(full.numel() == shard.numel() * getSize(), "cgx: ", name, "_compressed: the ", rs ? "input" : "output",
              " has ", full.numel(), " elements, expected world size (", getSize(), ") x ", rs ? "output" : "input",
              " (", shard.numel(), ")");
  TORCH_CHECK(bits >= 1 && (bits <= 8 || bits == kRawBits), "cgx: ", name, "_compressed: bits must be 1..8 or 32");
  TORCH_CHECK(engine_->nodes() == 1, "cgx: the compressed ", op_title(op), " supports a single node only");
  TORCH_CHECK(cfg_.inner_comm == CommType::kP2P, "cgx: the compressed ", op_title(op),
              " needs the P2P transport, not CGX_INNER_COMMUNICATOR_TYPE=", to_string(cfg_.inner_comm));
  RngParams rng;
  rng.stochastic = stochastic;
  rng.seed = seed >= 0 ? (uint64_t)seed : CompressionEnv::read().seed;
  return enqueue_cuda(rs ? c10d::OpType::_REDUCE_SCATTER_BASE : c10d::OpType::_ALLGATHER_BASE,
                      rs ? "cgx:reduce_scatter" : "cgx:all_gather", out, &in, [&](cudaStream_t s) {
                        engine_->sharded_cuda(op, in.data_ptr(), out.data_ptr(), dtype, shard.numel(), layers,
                                              average, bits, bucket_size, skip_incomplete, rng, s, overlapped);
                      });
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::engine_allreduce_cpu(at::Tensor& t, bool average, int bucket_idx) {
  // host tensors: queued to the worker thread in call order (reference: enqueue/runLoop,
  // ProcessGroupCGX.cc:300-339); the returned Work's future completes when the job is done, errors
  // are delivered through it
  {
    std::lock_guard<std::mutex> lk(mu_);
    ++seq_;
    if (!worker_) worker_ = std::make_unique<HostWorker>();
  }
  auto fut = c10::make_intrusive<c10::ivalue::Future>(c10::ListType::create(c10::TensorType::get()));
  at::Tensor tensor = t;
  const int dtype = to_cgx_dtype(t.scalar_type());
  // environment + layer table are captured NOW, on the caller's thread (functional.compression()
  // restores os.environ as soon as this returns)
  auto call = std::make_shared<AllreduceEngine::CpuCall>(engine_->prepare_cpu(tensor.numel(), bucket_idx));
  worker_->submit([this, fut, tensor, dtype, average, call]() mutable {
    try {
      engine_->allreduce_cpu_prepared(tensor.data_ptr(), dtype, *call, average);
      fut->markCompleted(at::IValue(std::vector<at::Tensor>{tensor}));
    } catch (...) {
      fut->setError(std::current_exception());
    }
  });
  return c10d::Work::create_from_future(fut);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::allreduce(std::vector<at::Tensor>& tensors,
                                                          const c10d::AllreduceOptions& opts) {
  TORCH_CHECK(tensors.size() == 1, "cgx: allreduce expects exactly one tensor");
  at::Tensor& t = tensors[0];
  if (eligible_for_engine(t, opts.reduceOp)) {
    const bool avg = opts.reduceOp == c10d::ReduceOp::AVG;
    return t.is_cuda() ? engine_allreduce(t, avg, -1) : engine_allreduce_cpu(t, avg, -1);
  }
  return delegate_for(t, "allreduce")->allreduce(tensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::allreduce_bucket(at::Tensor& tensor, int64_t bucket_idx,
                                                                 bool average) {
  c10d::ReduceOp op = average ? c10d::ReduceOp::AVG : c10d::ReduceOp::SUM;
  if (eligible_for_engine(tensor, op))
    return tensor.is_cuda() ? engine_allreduce(tensor, average, (int)bucket_idx)
                            : engine_allreduce_cpu(tensor, average, (int)bucket_idx);
  std::vector<at::Tensor> ts{tensor};
  c10d::AllreduceOptions o;
  if (average && !tensor.is_cuda()) {
    // Gloo has no AVG: pre-divide like the reference hook does
    tensor.div_(getSize());
    o.reduceOp = c10d::ReduceOp::SUM;
  } else {
    o.reduceOp = op;
  }
  return delegate_for(tensor, "allreduce")->allreduce(ts, o);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::allreduce_coalesced(std::vector<at::Tensor>& tensors,
                                                                    const c10d::AllreduceCoalescedOptions& opts) {
  TORCH_CHECK(!tensors.empty(), "cgx: allreduce_coalesced needs tensors");
  return delegate_for(tensors[0], "allreduce_coalesced")->allreduce_coalesced(tensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::broadcast(std::vector<at::Tensor>& tensors,
                                                          const c10d::BroadcastOptions& opts) {
  TORCH_CHECK(!tensors.empty(), "cgx: broadcast needs tensors");
  return delegate_for(tensors[0], "broadcast")->broadcast(tensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::reduce(std::vector<at::Tensor>& tensors,
                                                       const c10d::ReduceOptions& opts) {
  TORCH_CHECK(!tensors.empty(), "cgx: reduce needs tensors");
  return delegate_for(tensors[0], "reduce")->reduce(tensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::allgather(std::vector<std::vector<at::Tensor>>& outputTensors,
                                                          std::vector<at::Tensor>& inputTensors,
                                                          const c10d::AllgatherOptions& opts) {
  TORCH_CHECK(!inputTensors.empty(), "cgx: allgather needs tensors");
  return delegate_for(inputTensors[0], "allgather")->allgather(outputTensors, inputTensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::_allgather_base(at::Tensor& outputBuffer, at::Tensor& inputBuffer,
                                                                const c10d::AllgatherOptions& opts) {
  return delegate_for(inputBuffer, "_allgather_base")->_allgather_base(outputBuffer, inputBuffer, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::allgather_coalesced(
    std::vector<std::vector<at::Tensor>>& outputTensorLists, std::vector<at::Tensor>& inputTensors,
    const c10d::AllgatherOptions& opts) {
  TORCH_CHECK(!inputTensors.empty(), "cgx: allgather_coalesced needs tensors");
  return delegate_for(inputTensors[0], "allgather_coalesced")
      ->allgather_coalesced(outputTensorLists, inputTensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::allgather_into_tensor_coalesced(
    std::vector<at::Tensor>& outputs, std::vector<at::Tensor>& inputs, const c10d::AllgatherOptions& opts) {
  TORCH_CHECK(!inputs.empty(), "cgx: allgather_into_tensor_coalesced needs tensors");
  return delegate_for(inputs[0], "allgather_into_tensor_coalesced")
      ->allgather_into_tensor_coalesced(outputs, inputs, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::gather(std::vector<std::vector<at::Tensor>>& outputTensors,
                                                       std::vector<at::Tensor>& inputTensors,
                                                       const c10d::GatherOptions& opts) {
  TORCH_CHECK(!inputTensors.empty(), "cgx: gather needs tensors");
  return delegate_for(inputTensors[0], "gather")->gather(outputTensors, inputTensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::scatter(std::vector<at::Tensor>& outputTensors,
                                                        std::vector<std::vector<at::Tensor>>& inputTensors,
                                                        const c10d::ScatterOptions& opts) {
  TORCH_CHECK(!outputTensors.empty(), "cgx: scatter needs tensors");
  return delegate_for(outputTensors[0], "scatter")->scatter(outputTensors, inputTensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::reduce_scatter(std::vector<at::Tensor>& outputTensors,
                                                               std::vector<std::vector<at::Tensor>>& inputTensors,
                                                               const c10d::ReduceScatterOptions& opts) {
  TORCH_CHECK(!outputTensors.empty(), "cgx: reduce_scatter needs tensors");
  return delegate_for(outputTensors[0], "reduce_scatter")->reduce_scatter(outputTensors, inputTensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::_reduce_scatter_base(at::Tensor& outputBuffer,
                                                                     at::Tensor& inputBuffer,
                                                                     const c10d::ReduceScatterOptions& opts) {
  return delegate_for(inputBuffer, "_reduce_scatter_base")->_reduce_scatter_base(outputBuffer, inputBuffer, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::reduce_scatter_tensor_coalesced(
    std::vector<at::Tensor>& outputs, std::vector<at::Tensor>& inputs, const c10d::ReduceScatterOptions& opts) {
  TORCH_CHECK(!inputs.empty(), "cgx: reduce_scatter_tensor_coalesced needs tensors");
  return delegate_for(inputs[0], "reduce_scatter_tensor_coalesced")
      ->reduce_scatter_tensor_coalesced(outputs, inputs, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::alltoall_base(at::Tensor& outputBuffer, at::Tensor& inputBuffer,
                                                              std::vector<int64_t>& outputSplitSizes,
                                                              std::vector<int64_t>& inputSplitSizes,
                                                              const c10d::AllToAllOptions& opts) {
  return delegate_for(inputBuffer, "alltoall_base")
      ->alltoall_base(outputBuffer, inputBuffer, outputSplitSizes, inputSplitSizes, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::alltoall(std::vector<at::Tensor>& outputTensors,
                                                         std::vector<at::Tensor>& inputTensors,
                                                         const c10d::AllToAllOptions& opts) {
  TORCH_CHECK(!inputTensors.empty(), "cgx: alltoall needs tensors");
  return delegate_for(inputTensors[0], "alltoall")->alltoall(outputTensors, inputTensors, opts);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::send(std::vector<at::Tensor>& tensors, int dstRank, int tag) {
  TORCH_CHECK(!tensors.empty(), "cgx: send needs tensors");
  return delegate_for(tensors[0], "send")->send(tensors, dstRank, tag);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::recv(std::vector<at::Tensor>& tensors, int srcRank, int tag) {
  TORCH_CHECK(!tensors.empty(), "cgx: recv needs tensors");
  return delegate_for(tensors[0], "recv")->recv(tensors, srcRank, tag);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::recvAnysource(std::vector<at::Tensor>& tensors, int tag) {
  TORCH_CHECK(!tensors.empty(), "cgx: recvAnysource needs tensors");
  return delegate_for(tensors[0], "recvAnysource")->recvAnysource(tensors, tag);
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::barrier(const c10d::BarrierOptions& opts) {
  // A barrier must also drain this backend's own host worker and side stream.
  if (worker_) worker_->drain();
  if (cuda_ready_ && device_ >= 0) {
    c10::cuda::CUDAGuard g(device_);
    comm_stream_->synchronize();
    check_health();
  }
  const bool use_cuda = cuda_delegate_ && (opts.device.has_value() ? opts.device->is_cuda() : device_ >= 0);
  if (use_cuda) return cuda_delegate_->barrier(opts);
  TORCH_CHECK(cpu_delegate_, "cgx: no delegate backend available for barrier");
  return cpu_delegate_->barrier(opts);
}

int64_t ProcessGroupCGX::lanes() const { return engine_ && engine_->has_p2p() ? engine_->fused()->max_lanes() : 0; }

std::vector<int64_t> ProcessGroupCGX::stats() const {
  if (!engine_) return {0, 0, 0, 0, 0};
  const EngineStats& s = engine_->stats();
  return {(int64_t)s.calls, (int64_t)s.kernel_launches, (int64_t)s.elements, (int64_t)s.wire_bytes,
          (int64_t)s.raw_bytes};
}

void ProcessGroupCGX::reset_stats() {
  if (engine_) engine_->reset_stats();
}

void ProcessGroupCGX::enable_trace(bool on) {
  TORCH_CHECK(engine_ && engine_->has_p2p(), "cgx: enable_trace needs the P2P engine (call init_cuda first)");
  c10::cuda::CUDAGuard g(device_);
  engine_->fused()->enable_trace(on);
}

at::Tensor ProcessGroupCGX::read_trace() {
  TORCH_CHECK(engine_ && engine_->has_p2p(), "cgx: read_trace needs the P2P engine");
  c10::cuda::CUDAGuard g(device_);
  std::vector<uint64_t> v = engine_->fused()->read_trace();
  at::Tensor t = at::empty({(int64_t)v.size() / 8, 8}, at::kLong);
  std::memcpy(t.data_ptr(), v.data(), v.size() * sizeof(uint64_t));
  return t;
}

void ProcessGroupCGX::check_health() {
  const std::string msg = poll_failure();
  if (!msg.empty()) throw std::runtime_error(msg);
}

}  // namespace cgx

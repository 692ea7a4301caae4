#include "process_group_cgx.h"

#include <c10/cuda/CUDACachingAllocator.h>
#include <c10/cuda/CUDAGraphsC10Utils.h>
#include <c10/cuda/CUDAGuard.h>

#include <algorithm>
#include <cstring>

#include "../common/a2a.h"
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
    // the compressed all-to-all's cross-node chunks travel between any two ranks of the world
    if (engine_->nodes() > 1 && cuda_delegate_)
      engine_->attach_world(true, std::make_unique<C10dCommunicator>(cuda_delegate_, true, dev));
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

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::engine_allreduce(at::Tensor& t, bool average, int bucket_idx,
                                                                 std::optional<WireCodec> codec) {
  return enqueue_cuda(c10d::OpType::ALLREDUCE, "cgx:all_reduce", t, nullptr, [&](cudaStream_t s) {
    engine_->allreduce_cuda(t.data_ptr(), to_cgx_dtype(t.scalar_type()), t.numel(), average, bucket_idx, s,
                            /*overlapped=*/bucket_idx >= 0, codec);
  });
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::sharded_compressed(ShardedOp op, at::Tensor& out, at::Tensor& in,
                                                                   bool average, int bits, WireCodec codec,
                                                                   int bucket_size, bool skip_incomplete,
                                                                   bool stochastic,
                                                                   int64_t seed, bool overlapped,
                                                                   const std::vector<LayerSpec>& layers,
                                                                   const at::Tensor& out_scales) {
  const bool rs = op == ShardedOp::kReduceScatter;
  const char* name = op_name(op);
  const bool codes = out_scales.defined();
  TORCH_CHECK(in.is_cuda() && out.is_cuda(), "cgx: ", name, "_compressed needs CUDA tensors");
  TORCH_CHECK(in.device() == out.device(), "cgx: ", name, "_compressed: input and output on different devices");
  const int dtype = to_cgx_dtype(in.scalar_type());
  if (codes) {
    TORCH_CHECK(!rs, "cgx: output_scales is an all_gather output");
    TORCH_CHECK(codec != kMaxMin, "cgx: all_gather: output_scales needs bits=\"e4m3\" or \"e5m2\"");
    const at::ScalarType want = fp8_base(codec) == kE4M3 ? at::kFloat8_e4m3fn : at::kFloat8_e5m2;
    TORCH_CHECK(dtype >= 0 && out.scalar_type() == want, "cgx: all_gather: with output_scales the input must be ",
                "float32, float16 or bfloat16 and the output ", want, ", got ", in.scalar_type(), " and ",
                out.scalar_type());
    TORCH_CHECK(layers.empty(), "cgx: all_gather: output_scales takes no layer table (raw layers have no codes)");
  } else {
    TORCH_CHECK(dtype >= 0 && out.scalar_type() == in.scalar_type(), "cgx: ", name,
                "_compressed needs float32, float16 or bfloat16 tensors of one dtype, got ", in.scalar_type(), " and ",
                out.scalar_type());
  }
  TORCH_CHECK(in.is_contiguous() && out.is_contiguous(), "cgx: ", name, "_compressed needs contiguous tensors");
  const at::Tensor& full = rs ? in : out;
  const at::Tensor& shard = rs ? out : in;
  TORCH_CHECK(full.numel() == shard.numel() * getSize(), "cgx: ", name, "_compressed: the ", rs ? "input" : "output",
              " has ", full.numel(), " elements, expected world size (", getSize(), ") x ", rs ? "output" : "input",
              " (", shard.numel(), ")");
  TORCH_CHECK(bits >= 1 && (bits <= 8 || bits == kRawBits), "cgx: ", name, "_compressed: bits must be 1..8 or 32");
  TORCH_CHECK(codec == kMaxMin || (bits == 8 && (!stochastic || fp8_sr(codec))), "cgx: ", name,
              "_compressed: the FP8 formats use bits 8 and round to nearest (stochastically: the _sr formats)");
  RngParams rng;
  rng.stochastic = stochastic;
  rng.seed = seed >= 0 ? (uint64_t)seed : CompressionEnv::read().seed;
  // the codes output: one 8-bit layer whatever CGX_COMPRESSION_MINIMAL_SIZE says (a raw one has no codes)
  const std::vector<LayerSpec> table =
      codes ? std::vector<LayerSpec>{LayerSpec{0, (uint64_t)shard.numel(), 8, (uint32_t)std::max(1, bucket_size)}}
            : engine_->sharded_table(shard.numel(), layers, bits, bucket_size);
  if (codec != kMaxMin)
    for (const LayerSpec& l : table)
      TORCH_CHECK(l.bits == 8 || l.bits >= kRawBits, "cgx: ", name,
                  "_compressed: an FP8 format needs layers of bits 8 or 32, got ", l.bits);
  float* scales = nullptr;
  if (codes) {
    const int W = getSize();
    // every rank evaluates the same condition, so every rank refuses and none is left waiting
    TORCH_CHECK(local_size() >= W, "cgx: the compressed all_gather with output_scales runs on one node only ",
                "(CGX_LOCAL_SIZE ", local_size(), " < world size ", W, ")");
    const int64_t S = in.numel();
    TORCH_CHECK(bucket_size >= 1 && bucket_size <= (int)kMaxBlockElems && S % bucket_size == 0,
                "cgx: all_gather: output_scales needs 1 <= bucket_size <= ", kMaxBlockElems,
                " dividing the input's ", S, " elements, got ", bucket_size);
    TORCH_CHECK(out_scales.is_cuda() && out_scales.device() == out.device() && out_scales.scalar_type() == at::kFloat &&
                    out_scales.is_contiguous() && out_scales.numel() * bucket_size == out.numel(),
                "cgx: all_gather: output_scales must be a contiguous float32 tensor of ", out.numel() / bucket_size,
                " elements on ", out.device(), ", got ", out_scales.scalar_type(), " ", out_scales.sizes(), " on ",
                out_scales.device());
    scales = out_scales.data_ptr<float>();
    check_sharded_buffers(op, table, dtype, in.data_ptr(), out.data_ptr(), (uint64_t)S, getRank(), W, codec, scales);
  }
  return enqueue_cuda(rs ? c10d::OpType::_REDUCE_SCATTER_BASE : c10d::OpType::_ALLGATHER_BASE,
                      rs ? "cgx:reduce_scatter" : "cgx:all_gather", out, &in, [&](cudaStream_t s) {
                        if (codes) c10::cuda::CUDACachingAllocator::recordStream(out_scales.storage().data_ptr(), *comm_stream_);
                        // several nodes: the node partials / gathered shards, N x S elements
                        at::Tensor staging;
                        if (const int64_t n = engine_->sharded_staging_numel(shard.numel())) {
                          c10::cuda::CUDAStreamGuard sg(*comm_stream_);
                          staging = at::empty({n}, in.options());
                          c10::cuda::CUDACachingAllocator::recordStream(staging.storage().data_ptr(), *comm_stream_);
                        }
                        engine_->sharded(true, op, in.data_ptr(), out.data_ptr(),
                                         staging.defined() ? staging.data_ptr() : nullptr, dtype, shard.numel(), table,
                                         average, skip_incomplete, rng, s, overlapped, codec, scales);
                      });
}

namespace {

// per-rank element counts of one side of an all_to_all_single, from its dim-0 splits; `rows` are
// the rows of the side's tensor, or the entries of its index when `indexed`
std::vector<uint64_t> a2a_counts(int64_t rows, const std::vector<int64_t>& splits, int world, int64_t row,
                                 const char* side, bool indexed) {
  const std::string what = indexed ? std::string(side) + "_index" : std::string(side);
  const char* unit = indexed ? " entries" : " rows";
  std::vector<uint64_t> counts((size_t)world);
  if (splits.empty()) {
    TORCH_CHECK(rows % world == 0, "cgx: all_to_all: the ", what, " has ", rows, unit,
                ", not divisible by the world size ", world, " (give ", side, "_split_sizes)");
    for (auto& c : counts) c = (uint64_t)(rows / world * row);
    return counts;
  }
  TORCH_CHECK((int)splits.size() == world, "cgx: all_to_all: ", side, "_split_sizes has ", splits.size(),
              " entries, expected the world size ", world);
  int64_t sum = 0;
  for (int q = 0; q < world; ++q) {
    TORCH_CHECK(splits[q] >= 0, "cgx: all_to_all: ", side, "_split_sizes[", q, "] is negative (", splits[q], ")");
    sum += splits[q];
    counts[q] = (uint64_t)(splits[q] * row);
  }
  TORCH_CHECK(sum == rows, "cgx: all_to_all: ", side, "_split_sizes sums to ", sum, " but the ", what, " has ", rows,
              unit);
  return counts;
}

void check_a2a_index(const at::Tensor& index, const at::Tensor& like, const char* name) {
  if (!index.defined()) return;
  TORCH_CHECK(index.is_cuda() && index.device() == like.device(), "cgx: all_to_all: ", name,
              " must be on the device of the tensors (", like.device(), "), got ", index.device());
  TORCH_CHECK(index.scalar_type() == at::kLong, "cgx: all_to_all: ", name, " must be int64, got ", index.scalar_type());
  TORCH_CHECK(index.dim() == 1 && index.is_contiguous(), "cgx: all_to_all: ", name,
              " must be a contiguous 1-d tensor, got sizes ", index.sizes());
}

}  // namespace

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::all_to_all_compressed(at::Tensor& out, at::Tensor& in,
                                                                      const std::vector<int64_t>& out_splits,
                                                                      const std::vector<int64_t>& in_splits, int bits,
                                                                      WireCodec codec, int bucket_size, bool stochastic,
                                                                      int64_t seed,
                                                                      const at::Tensor& in_index,
                                                                      const at::Tensor& out_index,
                                                                      const at::Tensor& out_scales,
                                                                      const at::Tensor& gate,
                                                                      const at::Tensor& combine_out,
                                                                      const at::Tensor& in_scale) {
  TORCH_CHECK(in.is_cuda() && out.is_cuda(), "cgx: all_to_all needs CUDA tensors");
  TORCH_CHECK(in.device() == out.device(), "cgx: all_to_all: input and output on different devices");
  const int dtype = to_cgx_dtype(in.scalar_type());
  const bool codes = out_scales.defined();
  if (codes) {
    TORCH_CHECK(codec != kMaxMin, "cgx: all_to_all: output_scales needs bits=\"e4m3\" or \"e5m2\"");
    const at::ScalarType want = fp8_base(codec) == kE4M3 ? at::kFloat8_e4m3fn : at::kFloat8_e5m2;
    TORCH_CHECK(dtype >= 0 && out.scalar_type() == want, "cgx: all_to_all: with output_scales the input must be ",
                "float32, float16 or bfloat16 and the output ", want, ", got ", in.scalar_type(), " and ",
                out.scalar_type());
  } else {
    TORCH_CHECK(dtype >= 0 && out.scalar_type() == in.scalar_type(),
                "cgx: all_to_all needs float32, float16 or bfloat16 tensors of one dtype, got ", in.scalar_type(),
                " and ", out.scalar_type());
  }
  TORCH_CHECK(in.is_contiguous() && out.is_contiguous(), "cgx: all_to_all needs contiguous tensors");
  TORCH_CHECK(in.dim() >= 1 && out.dim() >= 1, "cgx: all_to_all needs tensors with at least one dimension");
  TORCH_CHECK(in.sizes().slice(1) == out.sizes().slice(1), "cgx: all_to_all: the input rows ", in.sizes().slice(1),
              " and the output rows ", out.sizes().slice(1), " differ");
  TORCH_CHECK(bits >= 1 && (bits <= 8 || bits == kRawBits), "cgx: all_to_all: bits must be 1..8 or 32");
  TORCH_CHECK(bucket_size >= 1, "cgx: all_to_all: bucket_size must be >= 1");
  TORCH_CHECK(codec == kMaxMin || (bits == 8 && (!stochastic || fp8_sr(codec))),
              "cgx: all_to_all: the FP8 codecs use bits 8 and round to nearest (stochastically: the _sr codecs)");
  const int W = getSize();
  // one node: the fused kernel's peers; several nodes: the cross-node stage's stream keys (a2a_rng_stream)
  const int max_world = local_size() >= W ? kMaxPeers : kA2aMaxWorld;
  TORCH_CHECK(W <= max_world, "cgx: all_to_all supports at most ", max_world, " ranks", local_size() >= W ? " on one node" : "");
  check_a2a_index(in_index, in, "input_index");
  check_a2a_index(out_index, out, "output_index");
  const bool ii = in_index.defined(), oi = out_index.defined();
  int64_t row = 1;
  for (int64_t d : in.sizes().slice(1)) row *= d;
  const bool combine = combine_out.defined();
  int64_t topk = 0;
  if (combine) {
    // the checks of cgx.all_to_all_combine, repeated for callers of the binding
    TORCH_CHECK_VALUE(!codes, "cgx: all_to_all_combine: a codes output (output_scales) has no combine");
    TORCH_CHECK_VALUE(oi, "cgx: all_to_all_combine needs an output_index");
    TORCH_CHECK_VALUE(gate.defined() && gate.scalar_type() == at::kFloat && gate.is_cuda() &&
                          gate.device() == out.device() && gate.is_contiguous() && gate.dim() == 2,
                      "cgx: all_to_all_combine: the gate must be a contiguous CUDA float32 tensor [T, k] on ",
                      out.device());
    topk = gate.size(1);
    TORCH_CHECK_VALUE(topk >= 1 && topk <= 32, "cgx: all_to_all_combine: k = ", topk, " is not in 1..32");
    const int64_t T = gate.size(0);
    TORCH_CHECK_VALUE(out_index.size(0) == T * topk && out.size(0) == T * topk,
                      "cgx: all_to_all_combine: output_index and the slots need T * k = ", T * topk,
                      " entries and rows, got ", out_index.size(0), " and ", out.size(0));
    TORCH_CHECK_VALUE(combine_out.scalar_type() == in.scalar_type() && combine_out.is_cuda() &&
                          combine_out.device() == out.device() && combine_out.is_contiguous() &&
                          combine_out.dim() >= 1 && combine_out.size(0) == T &&
                          combine_out.sizes().slice(1) == in.sizes().slice(1),
                      "cgx: all_to_all_combine: the output must be a contiguous ", in.scalar_type(), " tensor of ", T,
                      " rows like the input's on ", out.device());
  }
  const bool scaled = in_scale.defined();
  if (scaled) {
    // the checks of cgx.all_to_all_single's input_scale, repeated for callers of the binding
    TORCH_CHECK_VALUE(ii, "cgx: all_to_all: input_scale needs an input_index");
    TORCH_CHECK_VALUE(!codes, "cgx: all_to_all: input_scale has no codes output (output_scales)");
    TORCH_CHECK_VALUE(!combine, "cgx: all_to_all: input_scale has no combine (gate)");
    TORCH_CHECK_VALUE(in_scale.scalar_type() == at::kFloat && in_scale.is_cuda() && in_scale.device() == in.device() &&
                          in_scale.is_contiguous() && in_scale.dim() == 1 && in_scale.size(0) == in_index.size(0),
                      "cgx: all_to_all: input_scale must be a contiguous CUDA float32 vector of ", in_index.size(0),
                      " entries (one per input_index entry) on ", in.device(), ", got ", in_scale.scalar_type(), " ",
                      in_scale.sizes(), " on ", in_scale.device());
  }
  if (codes) {
    TORCH_CHECK(bucket_size <= (int)kMaxBlockElems && row % bucket_size == 0, "cgx: all_to_all: output_scales needs ",
                "bucket_size <= ", kMaxBlockElems, " dividing the row length ", row, ", got ", bucket_size);
    TORCH_CHECK(out_scales.is_cuda() && out_scales.device() == out.device() && out_scales.scalar_type() == at::kFloat &&
                    out_scales.is_contiguous() && out_scales.dim() == 2 && out_scales.size(0) == out.size(0) &&
                    out_scales.size(1) == row / bucket_size,
                "cgx: all_to_all: output_scales must be a contiguous float32 tensor of shape [", out.size(0), ", ",
                row / bucket_size, "] on ", out.device(), ", got ", out_scales.scalar_type(), " ", out_scales.sizes(),
                " on ", out_scales.device());
  }
  const std::vector<uint64_t> in_counts = a2a_counts(ii ? in_index.size(0) : in.size(0), in_splits, W, row, "input", ii);
  const std::vector<uint64_t> out_counts =
      a2a_counts(oi ? out_index.size(0) : out.size(0), out_splits, W, row, "output", oi);
  RngParams rng;
  rng.stochastic = stochastic;
  rng.seed = seed >= 0 ? (uint64_t)seed : CompressionEnv::read().seed;
  A2aRoute route;
  route.in_index = ii ? in_index.data_ptr<int64_t>() : nullptr;
  route.out_index = oi ? out_index.data_ptr<int64_t>() : nullptr;
  route.row = (uint64_t)row;
  route.in_rows = (uint64_t)in.size(0);
  route.out_rows = (uint64_t)out.size(0);
  if (combine) {
    route.combine_out = combine_out.data_ptr();
    route.gate = gate.data_ptr<float>();
    route.topk = (uint32_t)topk;
  }
  if (scaled) route.in_scale = in_scale.data_ptr<float>();
  const bool routed = ii || oi;
  float* scales = codes ? out_scales.data_ptr<float>() : nullptr;
  check_all_to_all(in.data_ptr(), out.data_ptr(), in_counts, out_counts, dtype, bits, codec, (uint32_t)bucket_size,
                   getRank(), W, routed ? &route : nullptr, scales);
  // the one place that decides where the rows are routed: inside the fused kernel when it can
  // address them, else around a plain call, which computes the same by definition
  const bool in_kernel = routed && engine_->routes_in_kernel(true, dtype, bits, (uint32_t)bucket_size, (uint64_t)row);
  return enqueue_cuda(c10d::OpType::ALLTOALL_BASE, "cgx:all_to_all", out, &in, [&](cudaStream_t s) {
    for (const at::Tensor* t : {&in_index, &out_index, &out_scales, &gate, &combine_out, &in_scale})
      if (t->defined()) c10::cuda::CUDACachingAllocator::recordStream(t->storage().data_ptr(), *comm_stream_);
    at::Tensor masks;
    if (combine && in_kernel) {
      // the arrival masks, zeroed on the comm stream inside the call, so a captured graph zeroes
      // them on every replay
      c10::cuda::CUDAStreamGuard sg(*comm_stream_);
      const int64_t segs = row / (int64_t)a2a_row_span(bits, (uint32_t)bucket_size, (int)dtype_size(dtype));
      masks = at::zeros({gate.size(0) * segs}, in.options().dtype(at::kInt));
      route.masks = reinterpret_cast<uint32_t*>(masks.data_ptr<int32_t>());
    }
    if (!routed || in_kernel) {
      engine_->all_to_all(true, in.data_ptr(), out.data_ptr(), in_counts, out_counts, dtype, bits, codec,
                          (uint32_t)bucket_size, rng, s, routed ? &route : nullptr, scales);
      return;
    }
    // the temporaries live on the comm stream only
    c10::cuda::CUDAStreamGuard sg(*comm_stream_);
    a2a_compose(*engine_, in, out, in_counts, out_counts, dtype, bits, codec, (uint32_t)bucket_size, rng, in_index,
                out_index, in_scale, out_scales, gate, combine_out, s);
  });
}

void a2a_compose(AllreduceEngine& engine, const at::Tensor& in, const at::Tensor& out,
                 const std::vector<uint64_t>& in_counts, const std::vector<uint64_t>& out_counts, int dtype, int bits,
                 WireCodec codec, uint32_t bucket, const RngParams& rng, const at::Tensor& in_index,
                 const at::Tensor& out_index, const at::Tensor& in_scale, const at::Tensor& out_scales,
                 const at::Tensor& gate, const at::Tensor& combine_out, cudaStream_t s) {
  const bool ii = in_index.defined(), oi = out_index.defined(), codes = out_scales.defined();
  int64_t row = 1;
  for (int64_t d : in.sizes().slice(1)) row *= d;
  const at::Tensor send = ii ? in.index_select(0, in_index) : in;
  // the scaled send: the selected rows times their scales, rounded as the fused kernel rounds them
  if (in_scale.defined())
    cuda_check(launch_scale_rows(send.data_ptr(), in_scale.data_ptr<float>(), dtype, (uint64_t)send.size(0),
                                 (uint64_t)row, s),
               "launch_scale_rows");
  std::vector<int64_t> recv_shape = out.sizes().vec();
  recv_shape[0] = oi ? out_index.size(0) : out.size(0);
  at::Tensor recv = oi ? at::empty(recv_shape, out.options()) : out;
  at::Tensor recv_scales = codes && oi ? at::empty({recv_shape[0], out_scales.size(1)}, out_scales.options()) : out_scales;
  engine.all_to_all(true, send.data_ptr(), recv.data_ptr(), in_counts, out_counts, dtype, bits, codec, bucket, rng, s,
                    nullptr, codes ? recv_scales.data_ptr<float>() : nullptr);
  if (oi && codes) {
    // the codes move as their bytes
    out.view(at::kByte).index_copy_(0, out_index, recv.view(at::kByte));
    out_scales.index_copy_(0, out_index, recv_scales);
  } else if (oi) {
    out.index_copy_(0, out_index, recv);
  }
  // the combine of the slots now in `out`, by the same arithmetic as the fused kernel's
  if (combine_out.defined())
    cuda_check(launch_combine_rows(out.data_ptr(), gate.data_ptr<float>(), combine_out.data_ptr(), dtype,
                                   (uint64_t)gate.size(0), (uint32_t)gate.size(1), (uint32_t)row, s),
               "launch_combine_rows");
}

c10::intrusive_ptr<c10d::Work> ProcessGroupCGX::engine_allreduce_cpu(at::Tensor& t, bool average, int bucket_idx,
                                                                     std::optional<WireCodec> codec) {
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
  if (codec) call->env.codec = *codec;
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
                                                                 bool average, std::optional<WireCodec> codec) {
  c10d::ReduceOp op = average ? c10d::ReduceOp::AVG : c10d::ReduceOp::SUM;
  if (eligible_for_engine(tensor, op))
    return tensor.is_cuda() ? engine_allreduce(tensor, average, (int)bucket_idx, codec)
                            : engine_allreduce_cpu(tensor, average, (int)bucket_idx, codec);
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

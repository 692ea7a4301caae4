// Python bindings: module torch_cgx_b200._C
//  * the c10d backend + the reference's pybind surface (register_layer,
//    set_quantization_bits, set_quantization_bucket_size;
//    /root/reference/src/ProcessGroupCGX.cc:837-857)
//  * planning / CPU oracle / standalone kernels for ops and tests
//  * LocalSraGroup: W virtual ranks of the fused kernels inside ONE process on
//    ONE GPU (W heaps, W streams) so the full protocol is testable on a single
//    device.
//  * LocalReducerGroup: W virtual ranks of the generic reducers (one host thread
//    each, loopback transport) on host memory or on ONE GPU.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <pybind11/chrono.h>
#include <torch/extension.h>

#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <thread>
#include <tuple>
#include <vector>

#include "comm/fd_channel.h"
#include "comm/loopback_communicator.h"
#include "common/block_ops.h"
#include "common/config.h"
#include "common/layers.h"
#include "common/plan.h"
#include "common/quant_error.h"
#include "common/sra_sim.h"
#include "kernels/launch.h"
#include "pg/comm_hook.h"
#include "pg/process_group_cgx.h"
#include "reduce/block_backend.h"
#include "reduce/reducers.h"

namespace py = pybind11;
using namespace cgx;

namespace {

using LayerTuple = std::tuple<int64_t, int64_t, int64_t, int64_t>;  // (elem_off, numel, bits, bucket)

std::vector<LayerSpec> to_layers(const std::vector<LayerTuple>& in) {
  std::vector<LayerSpec> out;
  out.reserve(in.size());
  for (const auto& t : in) {
    LayerSpec l;
    l.elem_off = (uint64_t)std::get<0>(t);
    l.numel = (uint64_t)std::get<1>(t);
    l.bits = (int)std::get<2>(t);
    l.bucket = (uint32_t)std::get<3>(t);
    out.push_back(l);
  }
  return out;
}

int cgx_dtype(const at::Tensor& t) {
  switch (t.scalar_type()) {
    case at::kFloat: return kF32;
    case at::kHalf: return kF16;
    case at::kBFloat16: return kBF16;
    default: TORCH_CHECK(false, "cgx: unsupported dtype ", t.scalar_type(), " (need float32/float16/bfloat16)");
  }
}

PlanOptions make_opts(int world, int lanes, int dtype, bool skip_incomplete, int64_t min_lane_elems) {
  PlanOptions o;
  o.world = world;
  o.lanes = lanes;
  o.dtype = dtype;
  o.skip_incomplete = skip_incomplete;
  o.min_lane_elems = (uint32_t)min_lane_elems;
  return o;
}

py::dict plan_to_dict(const Plan& p) {
  py::dict d;
  d["world"] = p.world;
  d["lanes"] = p.lanes;
  d["numel"] = p.numel;
  d["max_chunk_wire"] = p.max_chunk_wire;
  d["total_wire"] = p.total_wire;
  auto blocks = at::empty({(int64_t)p.blocks.size(), 5}, at::kLong);
  auto* bp = blocks.data_ptr<int64_t>();
  for (size_t i = 0; i < p.blocks.size(); ++i) {
    bp[i * 5 + 0] = p.blocks[i].elem_off;
    bp[i * 5 + 1] = block_n(p.blocks[i]);
    bp[i * 5 + 2] = block_bits(p.blocks[i]);
    bp[i * 5 + 3] = p.blocks[i].bucket;
    bp[i * 5 + 4] = p.blocks[i].wire_off;
  }
  d["blocks"] = blocks;
  auto items = at::empty({(int64_t)p.items.size(), 7}, at::kLong);
  auto* ip = items.data_ptr<int64_t>();
  for (size_t i = 0; i < p.items.size(); ++i) {
    ip[i * 7 + 0] = p.items[i].elem_off;
    ip[i * 7 + 1] = p.items[i].meta_off;
    ip[i * 7 + 2] = p.items[i].pay_off;
    ip[i * 7 + 3] = item_kind(p.items[i]);
    ip[i * 7 + 4] = item_lpb_log2(p.items[i]);
    ip[i * 7 + 5] = item_bits(p.items[i]);
    ip[i * 7 + 6] = item_n(p.items[i]);
  }
  d["items"] = items;  // rows: elem_off, meta_off, pay_off, kind, log2(bucket/8), bits, n
  d["item_first"] = std::vector<int64_t>(p.item_first.begin(), p.item_first.end());
  d["block_item_first"] = std::vector<int64_t>(p.block_item_first.begin(), p.block_item_first.end());
  d["slice_elems"] = p.slice_elems;
  d["uniform_bits"] = p.uniform_bits;
  d["lane_first"] = std::vector<int64_t>(p.lane_first.begin(), p.lane_first.end());
  d["chunk_wire_bytes"] = std::vector<int64_t>(p.chunk_wire_bytes.begin(), p.chunk_wire_bytes.end());
  d["chunk_elems"] = std::vector<int64_t>(p.chunk_elems.begin(), p.chunk_elems.end());
  return d;
}

RngParams make_rng(bool stochastic, uint64_t seed, uint32_t seq) {
  RngParams r;
  r.stochastic = stochastic;
  r.seed = seed;
  r.seq = seq;
  return r;
}

size_t wire_row_bytes(const Plan& p) { return ((size_t)p.max_chunk_wire + 255) / 256 * 256; }

// ---- CPU oracle ops -------------------------------------------------------
void py_sra_simulate(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, int lanes,
                     bool average, bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                     int64_t min_lane_elems) {
  TORCH_CHECK(!tensors.empty(), "need tensors");
  const int W = (int)tensors.size();
  const int dt = cgx_dtype(tensors[0]);
  std::vector<void*> bufs;
  for (auto& t : tensors) {
    TORCH_CHECK(t.device().is_cpu() && t.is_contiguous() && cgx_dtype(t) == dt, "sra_simulate: CPU contiguous tensors of one dtype");
    bufs.push_back(t.data_ptr());
  }
  Plan plan = build_plan(to_layers(layers), make_opts(W, lanes, dt, skip_incomplete, min_lane_elems));
  sra_simulate(plan, bufs, average ? 1.0f / (float)W : 1.0f, make_rng(stochastic, seed, seq));
}

void py_oneshot_simulate(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, int lanes,
                         bool average, bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                         int64_t min_lane_elems) {
  TORCH_CHECK(!tensors.empty(), "need tensors");
  const int W = (int)tensors.size();
  const int dt = cgx_dtype(tensors[0]);
  std::vector<void*> bufs;
  for (auto& t : tensors) {
    TORCH_CHECK(t.device().is_cpu() && t.is_contiguous() && cgx_dtype(t) == dt, "oneshot_simulate: CPU contiguous tensors");
    bufs.push_back(t.data_ptr());
  }
  Plan plan = build_plan(to_layers(layers), make_opts(1, lanes, dt, skip_incomplete, min_lane_elems));
  oneshot_simulate(plan, bufs, average ? 1.0f / (float)W : 1.0f, make_rng(stochastic, seed, seq));
}

// Argument checks of the sharded simulators: one CPU contiguous input and output per rank, all of
// the inputs' dtype, the full buffers of W * S elements and the shards of S. Returns S, the end of
// the shard table.
uint64_t check_sharded_simulate(ShardedOp op, const std::vector<at::Tensor>& inputs,
                                const std::vector<at::Tensor>& outputs, const std::vector<LayerSpec>& shard_layers) {
  const bool rs = op == ShardedOp::kReduceScatter;
  TORCH_CHECK(!inputs.empty() && inputs.size() == outputs.size(), op_name(op),
              "_simulate: one input and one output per rank");
  const uint64_t W = inputs.size(), S = shard_elems(shard_layers);
  const int dt = cgx_dtype(inputs[0]);
  for (size_t r = 0; r < W; ++r) {
    const at::Tensor &i = inputs[r], &o = outputs[r];
    TORCH_CHECK(i.device().is_cpu() && o.device().is_cpu() && i.is_contiguous() && o.is_contiguous() &&
                    cgx_dtype(i) == dt && cgx_dtype(o) == dt && (uint64_t)i.numel() == (rs ? S * W : S) &&
                    (uint64_t)o.numel() == (rs ? S : S * W),
                op_name(op), "_simulate: CPU contiguous tensors of one dtype, ",
                rs ? "inputs of W * S and outputs of S elements" : "inputs of S and outputs of W * S elements");
  }
  return S;
}

void py_reduce_scatter_simulate(const std::vector<at::Tensor>& inputs, std::vector<at::Tensor> outputs,
                                const std::vector<LayerTuple>& shard_layers, int lanes, bool average,
                                bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                                int64_t min_lane_elems) {
  const auto shard = to_layers(shard_layers);
  const uint64_t S = check_sharded_simulate(ShardedOp::kReduceScatter, inputs, outputs, shard);
  const int W = (int)inputs.size();
  const int dt = cgx_dtype(inputs[0]);
  std::vector<const void*> in;
  std::vector<void*> out;
  for (int r = 0; r < W; ++r) {
    in.push_back(inputs[r].data_ptr());
    out.push_back(outputs[r].data_ptr());
  }
  Plan plan = build_plan(replicate(shard, W, S), make_opts(W, lanes, dt, skip_incomplete, min_lane_elems));
  reduce_scatter_simulate(plan, in, out, S, average ? 1.0f / (float)W : 1.0f, make_rng(stochastic, seed, seq));
}

// All-gather oracle (ag_kernel): shard q is one quantization round trip (roundtrip_simulate) of
// in_q placed at q * S, through copy q of the replicated table and rank q's publish stream (phase
// 1, the SRA's requantization), so the RNG counters are the kernel's element indices. Every output
// gets the same bytes.
void py_all_gather_simulate(const std::vector<at::Tensor>& inputs, std::vector<at::Tensor> outputs,
                            const std::vector<LayerTuple>& shard_layers, bool stochastic, uint64_t seed,
                            uint32_t seq) {
  const auto shard = to_layers(shard_layers);
  const uint64_t S = check_sharded_simulate(ShardedOp::kAllGather, inputs, outputs, shard);
  const int W = (int)inputs.size();
  const int dt = cgx_dtype(inputs[0]);
  const auto layers = replicate(shard, W, S);
  const size_t es = (size_t)dtype_size(dt), per_copy = shard_layers.size();
  uint8_t* out0 = static_cast<uint8_t*>(outputs[0].data_ptr());
  for (int q = 0; q < W; ++q) {
    std::memcpy(out0 + (size_t)q * S * es, inputs[q].data_ptr(), S * es);
    const std::vector<LayerSpec> copy(layers.begin() + (ptrdiff_t)(q * per_copy),
                                      layers.begin() + (ptrdiff_t)((q + 1) * per_copy));
    roundtrip_simulate(build_plan(copy, make_opts(1, 1, dt, false, 1 << 30)), out0, 1.0f,
                       make_rng(stochastic, seed, seq), q, 1);
  }
  for (int r = 1; r < W; ++r) std::memcpy(outputs[r].data_ptr(), out0, S * W * es);
}

// quantize `t` through the plan; returns uint8 wire tensor [world, row_bytes]
at::Tensor py_quantize(const at::Tensor& t, const std::vector<LayerTuple>& layers, int world, int lanes,
                       bool skip_incomplete, float prescale, bool stochastic, uint64_t seed, uint32_t seq,
                       int rank, int phase, int64_t min_lane_elems) {
  TORCH_CHECK(t.is_contiguous(), "quantize: tensor must be contiguous");
  const int dt = cgx_dtype(t);
  Plan plan = build_plan(to_layers(layers), make_opts(world, lanes, dt, skip_incomplete, min_lane_elems));
  const size_t row = wire_row_bytes(plan);
  RngKey key = make_rng_key(make_rng(stochastic, seed, seq), rank, phase);
  if (t.device().is_cpu()) {
    at::Tensor wire = at::zeros({(int64_t)world, (int64_t)row}, at::kByte);
    std::vector<float> acc(kMaxBlockElems);
    for (int c = 0; c < world; ++c)
      for (uint32_t b = plan.chunk_begin(c); b < plan.chunk_end(c); ++b) {
        const BlockDesc& d = plan.blocks[b];
        cpu::load_block(t.data_ptr(), dt, d, prescale, acc.data());
        cpu::quantize_block(acc.data(), dt, d, wire.data_ptr<uint8_t>() + (size_t)c * row + d.wire_off, key, b);
      }
    return wire;
  }
  c10::cuda::CUDAGuard g(t.device());
  auto stream = c10::cuda::getCurrentCUDAStream();
  at::Tensor wire = at::zeros({(int64_t)world, (int64_t)row}, t.options().dtype(at::kByte));
  at::Tensor ditems = at::empty({(int64_t)(plan.items.size() * sizeof(WarpItem) + 16)}, t.options().dtype(at::kByte));
  cuda_check(cudaMemcpyAsync(ditems.data_ptr(), plan.items.data(), plan.items.size() * sizeof(WarpItem),
                             cudaMemcpyHostToDevice, stream),
             "upload items");
  for (int c = 0; c < world; ++c) {
    ItemKernelArgs a;
    a.items = (const WarpItem*)ditems.data_ptr();
    a.first = plan.item_first[(size_t)c * plan.lanes];
    a.count = plan.item_first[(size_t)(c + 1) * plan.lanes] - a.first;
    a.dtype = dt;
    a.slice_elems = (int)plan.slice_elems;
    a.uniform_bits = plan.uniform_bits;
    cuda_check(launch_quantize_items(a, t.data_ptr(), wire.data_ptr<uint8_t>() + (size_t)c * row, prescale, key, stream),
               "quantize_items");
  }
  return wire;
}

// inverse of py_quantize: decode `wire` into a tensor shaped like `like`
at::Tensor py_dequantize(const at::Tensor& wire, const at::Tensor& like, const std::vector<LayerTuple>& layers,
                         int world, int lanes, bool skip_incomplete, int64_t min_lane_elems) {
  const int dt = cgx_dtype(like);
  Plan plan = build_plan(to_layers(layers), make_opts(world, lanes, dt, skip_incomplete, min_lane_elems));
  const size_t row = wire_row_bytes(plan);
  TORCH_CHECK(wire.is_contiguous() && wire.scalar_type() == at::kByte && (size_t)wire.numel() == row * (size_t)world,
              "dequantize: wire tensor has the wrong shape");
  at::Tensor out = at::zeros_like(like);
  if (like.device().is_cpu()) {
    for (int c = 0; c < world; ++c)
      for (uint32_t b = plan.chunk_begin(c); b < plan.chunk_end(c); ++b) {
        const BlockDesc& d = plan.blocks[b];
        cpu::decode_block_store(wire.data_ptr<uint8_t>() + (size_t)c * row + d.wire_off, dt, d, out.data_ptr());
      }
    return out;
  }
  c10::cuda::CUDAGuard g(like.device());
  auto stream = c10::cuda::getCurrentCUDAStream();
  at::Tensor ditems = at::empty({(int64_t)(plan.items.size() * sizeof(WarpItem) + 16)}, like.options().dtype(at::kByte));
  cuda_check(cudaMemcpyAsync(ditems.data_ptr(), plan.items.data(), plan.items.size() * sizeof(WarpItem),
                             cudaMemcpyHostToDevice, stream),
             "upload items");
  for (int c = 0; c < world; ++c) {
    ItemKernelArgs a;
    a.items = (const WarpItem*)ditems.data_ptr();
    a.first = plan.item_first[(size_t)c * plan.lanes];
    a.count = plan.item_first[(size_t)(c + 1) * plan.lanes] - a.first;
    a.dtype = dt;
    a.slice_elems = (int)plan.slice_elems;
    a.uniform_bits = plan.uniform_bits;
    cuda_check(launch_dequantize_items(a, wire.data_ptr<uint8_t>() + (size_t)c * row, out.data_ptr(), stream),
               "dequantize_items");
  }
  return out;
}

// ---- pre-planned codec: the kernels alone, no per-call planning or allocation ----------------
// (kernel microbenchmarks, and users who quantize the same layout repeatedly)
class PreparedCodec {
 public:
  PreparedCodec(const std::vector<LayerTuple>& layers, at::ScalarType dtype, int64_t device, bool skip_incomplete) {
    at::Tensor probe = at::empty({0}, at::TensorOptions().dtype(dtype));
    dt_ = cgx_dtype(probe);
    plan_ = build_plan(to_layers(layers), make_opts(1, 1, dt_, skip_incomplete, 1 << 30));
    c10::cuda::CUDAGuard g((c10::DeviceIndex)device);
    items_ = at::empty({(int64_t)(plan_.items.size() * sizeof(WarpItem) + 16)},
                       at::TensorOptions().dtype(at::kByte).device(at::kCUDA, device));
    cuda_check(cudaMemcpy(items_.data_ptr(), plan_.items.data(), plan_.items.size() * sizeof(WarpItem),
                          cudaMemcpyHostToDevice),
               "upload items");
  }
  int64_t wire_bytes() const { return (int64_t)wire_row_bytes(plan_); }
  int64_t numel() const { return (int64_t)plan_.numel; }
  int64_t num_items() const { return (int64_t)plan_.items.size(); }
  void quantize(const at::Tensor& x, at::Tensor& wire, double prescale, bool stochastic, uint64_t seed, uint32_t seq) {
    check(x, wire);
    c10::cuda::CUDAGuard g(x.device());
    cuda_check(launch_quantize_items(args(), x.data_ptr(), wire.data_ptr<uint8_t>(), (float)prescale,
                                     make_rng_key(make_rng(stochastic, seed, seq), 0, 0),
                                     c10::cuda::getCurrentCUDAStream()),
               "quantize_items");
  }
  void dequantize(const at::Tensor& wire, at::Tensor& out) {
    check(out, wire);
    c10::cuda::CUDAGuard g(out.device());
    cuda_check(launch_dequantize_items(args(), wire.data_ptr<uint8_t>(), out.data_ptr(),
                                       c10::cuda::getCurrentCUDAStream()),
               "dequantize_items");
  }

 private:
  void check(const at::Tensor& x, const at::Tensor& wire) const {
    TORCH_CHECK(x.is_cuda() && x.is_contiguous() && cgx_dtype(x) == dt_ && (uint64_t)x.numel() == plan_.numel,
                "PreparedCodec: tensor does not match the prepared layout");
    TORCH_CHECK(wire.is_cuda() && wire.is_contiguous() && wire.scalar_type() == at::kByte &&
                    (size_t)wire.numel() >= wire_row_bytes(plan_),
                "PreparedCodec: wire buffer too small");
  }
  ItemKernelArgs args() const {
    ItemKernelArgs a;
    a.items = (const WarpItem*)items_.data_ptr();
    a.first = 0;
    a.count = (uint32_t)plan_.items.size();
    a.dtype = dt_;
    a.slice_elems = (int)plan_.slice_elems;
    a.uniform_bits = plan_.uniform_bits;
    return a;
  }
  Plan plan_;
  int dt_ = kF32;
  at::Tensor items_;
};

// ---- single-process multi-rank harness --------------------------------------
class LocalSraGroup {
 public:
  LocalSraGroup(int world, int lanes, int64_t slot_bytes, int64_t timeout_ms, int64_t min_lane_elems)
      : world_(world) {
    TORCH_CHECK(world >= 1 && world <= kMaxPeers, "bad world size");
    HeapLayout layout = HeapLayout::make(world, lanes, (size_t)slot_bytes, (size_t)slot_bytes);
    for (int r = 0; r < world; ++r) heaps_.push_back(std::make_unique<SymmetricHeap>(r, world, layout));
    std::vector<SymmetricHeap*> all;
    for (auto& h : heaps_) all.push_back(h.get());
    for (auto& h : heaps_) h->connect_local(all);
    for (int r = 0; r < world; ++r) {
      fused_.push_back(std::make_unique<FusedSra>(heaps_[r].get(), lanes, timeout_ms, (uint32_t)min_lane_elems));
      streams_.push_back(c10::cuda::getStreamFromPool(false));
    }
  }

  // in-place allreduce of W same-device tensors, one per virtual rank
  void allreduce_oneshot(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, bool average,
                         bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq) {
    run(std::move(tensors), layers, average, skip_incomplete, stochastic, seed, seq, true);
  }
  void allreduce(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, bool average,
                 bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq) {
    run(std::move(tensors), layers, average, skip_incomplete, stochastic, seed, seq, false);
  }
  // fault injection: virtual rank `absent` never launches its kernel (a dead / stuck peer)
  void allreduce_with_absent_rank(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers,
                                  int absent) {
    run(std::move(tensors), layers, false, false, false, 0, 1, false, absent);
  }
  void abort_all() {
    for (auto& h : heaps_) h->request_abort(true);
  }
  std::string status(int r) { return fused_[r]->status_message(); }
  void clear() {
    for (auto& f : fused_) f->clear_status();
  }
  void run(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, bool average,
           bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq, bool oneshot, int absent = -1) {
    TORCH_CHECK((int)tensors.size() == world_, "need one tensor per virtual rank");
    const int dt = cgx_dtype(tensors[0]);
    for (const at::Tensor& t : tensors)
      TORCH_CHECK(t.is_cuda() && t.is_contiguous() && cgx_dtype(t) == dt, "bad tensor");
    const auto specs = to_layers(layers);
    const RngParams rng = make_rng(stochastic, seed, seq);
    const float ps = average ? 1.0f / (float)world_ : 1.0f;
    std::vector<const DevicePlan*> plans(world_);
    fork_join(
        [&](int r) {
          plans[r] = oneshot ? fused_[r]->prepare_oneshot(specs, dt, skip_incomplete, streams_[r].stream())
                             : fused_[r]->prepare(specs, dt, skip_incomplete, streams_[r].stream());
          TORCH_CHECK(plans[r] != nullptr, "plan does not fit the heap slots (raise slot_bytes)");
        },
        [&](int r) {
          if (r == absent) return;
          if (oneshot)
            fused_[r]->run_oneshot(*plans[r], tensors[r].data_ptr(), ps, rng, streams_[r].stream());
          else
            fused_[r]->run(*plans[r], tensors[r].data_ptr(), ps, rng, streams_[r].stream());
        });
  }

  // reduce-scatter: inputs[r] holds W * S elements of virtual rank r, outputs[r] receives shard r
  void reduce_scatter(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs,
                      const std::vector<LayerTuple>& shard_layers, bool average, bool skip_incomplete,
                      bool stochastic, uint64_t seed, uint32_t seq) {
    sharded(ShardedOp::kReduceScatter, inputs, outputs, shard_layers, average, skip_incomplete, stochastic, seed, seq);
  }
  // all-gather: inputs[r] holds virtual rank r's shard of S elements, outputs[r] receives W * S
  void all_gather(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs,
                  const std::vector<LayerTuple>& shard_layers, bool stochastic, uint64_t seed, uint32_t seq) {
    sharded(ShardedOp::kAllGather, inputs, outputs, shard_layers, false, false, stochastic, seed, seq);
  }
  void check() {
    for (auto& f : fused_) f->check_status();
  }
  int64_t lanes_used(const std::vector<LayerTuple>& layers, const at::Tensor& like, bool skip_incomplete) {
    auto* dp = fused_[0]->prepare(to_layers(layers), cgx_dtype(like), skip_incomplete,
                                  c10::cuda::getCurrentCUDAStream().stream());
    return dp ? dp->plan.lanes : -1;
  }

 private:
  // Every virtual rank's stream starts after the caller's current stream and runs prepare(r) (plan
  // builds and uploads), then launch(r); the caller's stream waits for all of them.
  template <class Prepare, class Launch>
  void fork_join(Prepare&& prepare, Launch&& launch) {
    auto cur = c10::cuda::getCurrentCUDAStream();
    at::cuda::CUDAEvent ready(cudaEventDisableTiming);
    ready.record(cur);
    bool fresh_plan = false;
    for (int r = 0; r < world_; ++r) {
      ready.block(streams_[r]);
      const size_t before = fused_[r]->num_plans();
      prepare(r);
      fresh_plan = fresh_plan || fused_[r]->num_plans() != before;
    }
    // make sure every plan upload has landed before any virtual rank starts spinning
    if (fresh_plan)
      for (int r = 0; r < world_; ++r) streams_[r].synchronize();
    for (int r = 0; r < world_; ++r) launch(r);
    for (int r = 0; r < world_; ++r) {
      at::cuda::CUDAEvent done(cudaEventDisableTiming);
      done.record(streams_[r]);
      done.block(cur);
    }
  }

  void sharded(ShardedOp op, std::vector<at::Tensor>& inputs, std::vector<at::Tensor>& outputs,
               const std::vector<LayerTuple>& shard_layers, bool average, bool skip_incomplete, bool stochastic,
               uint64_t seed, uint32_t seq) {
    const bool rs = op == ShardedOp::kReduceScatter;
    TORCH_CHECK((int)inputs.size() == world_ && (int)outputs.size() == world_,
                "need one input and one output per virtual rank");
    const int dt = cgx_dtype(inputs[0]);
    for (int r = 0; r < world_; ++r) {
      for (const at::Tensor* t : {&inputs[r], &outputs[r]})
        TORCH_CHECK(t->is_cuda() && t->is_contiguous() && cgx_dtype(*t) == dt, "bad tensor");
      const at::Tensor &full = rs ? inputs[r] : outputs[r], &shard = rs ? outputs[r] : inputs[r];
      TORCH_CHECK(full.numel() == shard.numel() * world_,
                  rs ? "inputs must hold W x the output elements" : "outputs must hold W x the input elements");
    }
    const auto specs = to_layers(shard_layers);
    // streams r and r + 8 share a hardware queue (CUDA_DEVICE_MAX_CONNECTIONS = 8): with two kernels
    // per virtual rank, rank r + 8's first one would wait behind rank r's second, which waits for it
    TORCH_CHECK(world_ <= 8 || fused_[0]->rs_windows(specs, dt, skip_incomplete, 0).size() <= 1, "LocalSraGroup.",
                op_name(op), ": more than 8 virtual ranks need the shard to fit one window (raise slot_bytes)");
    const RngParams rng = make_rng(stochastic, seed, seq);
    const float ps = average ? 1.0f / (float)world_ : 1.0f;
    fork_join([&](int r) { fused_[r]->prepare_sharded(specs, dt, skip_incomplete, streams_[r].stream()); },
              [&](int r) {
                fused_[r]->sharded(op, specs, dt, skip_incomplete, inputs[r].data_ptr(), outputs[r].data_ptr(),
                                   (uint64_t)(rs ? outputs[r] : inputs[r]).numel(), ps, rng, streams_[r].stream());
              });
  }

  int world_;
  std::vector<std::unique_ptr<SymmetricHeap>> heaps_;
  std::vector<std::unique_ptr<FusedSra>> fused_;
  std::vector<c10::cuda::CUDAStream> streams_;
};

// W virtual ranks of one generic reducer (make_reducer), each with its own Reducer, BlockBackend,
// stream and host thread, connected by the loopback transport. CPU tensors run the host backend,
// tensors of one CUDA device the device backend: the same reducer code on both, in one process.
class LocalReducerGroup {
 public:
  LocalReducerGroup(int world, const std::string& kind, int64_t timeout_ms) : hub_(world, timeout_ms) {
    TORCH_CHECK(world >= 1 && world <= kMaxPeers, "LocalReducerGroup: world must be 1..", kMaxPeers, ", got ", world);
    if (kind == "SRA")
      kind_ = ReductionType::kSRA;
    else if (kind == "RING")
      kind_ = ReductionType::kRing;
    else if (kind == "ALLTOALL")
      kind_ = ReductionType::kAllToAll;
    else
      TORCH_CHECK(false, "LocalReducerGroup: kind must be SRA, RING or ALLTOALL, got ", kind);
    last_sent_.assign((size_t)world, 0);
  }
  ~LocalReducerGroup() {
    // the device reducers free their scratch on the device they allocated it on
    std::optional<c10::cuda::CUDAGuard> g;
    if (device_ >= 0) g.emplace((c10::DeviceIndex)device_);
    cuda_.clear();
  }

  // in-place allreduce of one tensor per virtual rank; the prescale is 1/W when averaging
  void allreduce(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, bool average,
                 bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq) {
    const auto specs = to_layers(layers);
    const RngParams rng = make_rng(stochastic, seed, seq);
    const float prescale = average ? 1.0f / (float)hub_.world() : 1.0f;
    run(tensors, [&](Reducer& red, void* data, int dt, cudaStream_t s) {
      red.allreduce(data, dt, specs, skip_incomplete, prescale, rng, s);
    });
  }
  void broadcast_compressed(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, int root,
                            bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq) {
    TORCH_CHECK(root >= 0 && root < hub_.world(), "LocalReducerGroup: bad root ", root);
    const auto specs = to_layers(layers);
    const RngParams rng = make_rng(stochastic, seed, seq);
    run(tensors, [&](Reducer& red, void* data, int dt, cudaStream_t s) {
      red.broadcast_compressed(data, dt, specs, skip_incomplete, root, rng, s);
    });
  }
  // bytes each rank's reducer counted as sent during the last call
  std::vector<int64_t> bytes_sent() const { return last_sent_; }
  void set_recording(bool on) { record_ = on; }
  // the messages of the last call (recording on): (exchange index, src, dst, uint8 CPU tensor)
  std::vector<std::tuple<int64_t, int, int, at::Tensor>> messages() const {
    std::vector<std::tuple<int64_t, int, int, at::Tensor>> out;
    for (const auto& m : hub_.messages()) {
      at::Tensor t = at::empty({(int64_t)m.bytes.size()}, at::kByte);
      if (!m.bytes.empty()) std::memcpy(t.data_ptr(), m.bytes.data(), m.bytes.size());
      out.emplace_back(m.exchange, m.src, m.dst, t);
    }
    return out;
  }

 private:
  struct Rank {
    std::unique_ptr<LoopbackCommunicator> comm;
    std::unique_ptr<BlockBackend> ops;
    std::unique_ptr<Reducer> red;  // declared last: released first, its scratch through `ops`
  };

  std::vector<Rank>& ranks(bool cuda) {
    std::vector<Rank>& v = cuda ? cuda_ : cpu_;
    if (v.empty())
      for (int r = 0; r < hub_.world(); ++r) {
        Rank k;
        k.comm = std::make_unique<LoopbackCommunicator>(&hub_, r, cuda);
        k.ops = cuda ? make_cuda_block_backend() : make_cpu_block_backend();
        k.red = make_reducer(kind_, k.comm.get(), k.ops.get());
        v.push_back(std::move(k));
      }
    return v;
  }

  template <class F>
  void run(const std::vector<at::Tensor>& tensors, F&& op) {
    const int W = hub_.world();
    TORCH_CHECK((int)tensors.size() == W, "LocalReducerGroup: need one tensor per virtual rank (", W, "), got ",
                tensors.size());
    const int dt = cgx_dtype(tensors[0]);
    const bool cuda = tensors[0].is_cuda();
    for (const at::Tensor& t : tensors)
      TORCH_CHECK(t.is_contiguous() && cgx_dtype(t) == dt && t.numel() == tensors[0].numel() &&
                      t.device() == tensors[0].device(),
                  "LocalReducerGroup: contiguous tensors of one dtype, size and device");
    TORCH_CHECK(cuda || tensors[0].device().is_cpu(), "LocalReducerGroup: CPU or CUDA tensors");
    if (cuda) {
      const int dev = tensors[0].device().index();
      TORCH_CHECK(device_ < 0 || device_ == dev, "LocalReducerGroup: all calls use one device (", device_, ")");
      device_ = dev;
    }
    c10::cuda::OptionalCUDAGuard guard;
    if (cuda) {
      guard.set_index((c10::DeviceIndex)device_);
      if (streams_.empty())
        for (int r = 0; r < W; ++r) streams_.push_back(c10::cuda::getStreamFromPool(false, (c10::DeviceIndex)device_));
      // every virtual rank starts after the work that produced its input
      at::cuda::CUDAEvent ready(cudaEventDisableTiming);
      ready.record(c10::cuda::getCurrentCUDAStream());
      for (auto& s : streams_) ready.block(s);
    }
    std::vector<Rank>& rk = ranks(cuda);
    std::vector<uint64_t> before(W);
    for (int r = 0; r < W; ++r) before[r] = rk[r].red->bytes_sent();
    hub_.reset(record_);
    {
      py::gil_scoped_release nogil;
      std::vector<std::thread> threads;
      for (int r = 0; r < W; ++r)
        threads.emplace_back([&, r] {
          try {
            c10::cuda::OptionalCUDAGuard g;
            cudaStream_t s = nullptr;
            if (cuda) {
              g.set_index((c10::DeviceIndex)device_);
              s = streams_[r].stream();
            }
            op(*rk[r].red, tensors[r].data_ptr(), dt, s);
            if (cuda) cuda_check(cudaStreamSynchronize(s), "LocalReducerGroup: synchronise a virtual rank");
          } catch (const std::exception& e) {
            hub_.fail("rank " + std::to_string(r) + ": " + e.what());
          } catch (...) {
            hub_.fail("rank " + std::to_string(r) + ": unknown exception");
          }
          hub_.finish(r);
        });
      for (auto& t : threads) t.join();
      // a rank that threw skipped its own synchronise: nothing it queued may still write the caller's
      // tensors or the scratch once this returns
      if (cuda)
        for (int r = 0; r < W; ++r) {
          const cudaError_t err = cudaStreamSynchronize(streams_[r].stream());
          if (err != cudaSuccess)
            hub_.fail("rank " + std::to_string(r) + ": synchronise after the call: " + cudaGetErrorString(err));
        }
    }
    for (int r = 0; r < W; ++r) last_sent_[r] = (int64_t)(rk[r].red->bytes_sent() - before[r]);
    TORCH_CHECK(!hub_.failed(), "LocalReducerGroup: ", hub_.failure());
  }

  LoopbackHub hub_;
  ReductionType kind_ = ReductionType::kSRA;
  bool record_ = false;
  int device_ = -1;
  std::vector<c10::cuda::CUDAStream> streams_;
  std::vector<Rank> cpu_, cuda_;
  std::vector<int64_t> last_sent_;
};

// ---- ResNet residual join: every operand like `ref` (device, dtype, sizes, strides), all dense ----
void check_join_operand(const at::Tensor& ref, const at::Tensor& t, const char* op, const char* name) {
  TORCH_CHECK(t.is_cuda(), op, ": ", name, " must be a CUDA tensor, got ", t.device());
  TORCH_CHECK(t.device() == ref.device(), op, ": ", name, " is on ", t.device(), ", the others on ", ref.device());
  TORCH_CHECK(t.scalar_type() == ref.scalar_type(), op, ": ", name, " is ", t.scalar_type(), ", the others ",
              ref.scalar_type());
  TORCH_CHECK(t.sizes() == ref.sizes(), op, ": ", name, " has sizes ", t.sizes(), ", the others ", ref.sizes());
  TORCH_CHECK(t.strides() == ref.strides(), op, ": ", name, " has strides ", t.strides(), ", the others ",
              ref.strides());
  TORCH_CHECK(t.is_non_overlapping_and_dense(), op, ": ", name, " must be non-overlapping and dense (strides ",
              t.strides(), ")");
}

at::Tensor py_residual_relu_forward(const at::Tensor& a, const at::Tensor& b) {
  check_join_operand(a, a, "residual_relu_forward", "a");
  check_join_operand(a, b, "residual_relu_forward", "b");
  const int dt = cgx_dtype(a);
  c10::cuda::CUDAGuard g(a.device());
  at::Tensor y = at::empty_like(a);  // dense input: same strides
  cuda_check(launch_residual_relu_forward(a.data_ptr(), b.data_ptr(), y.data_ptr(), dt, (uint64_t)a.numel(),
                                          c10::cuda::getCurrentCUDAStream()),
             "residual_relu_forward");
  return y;
}

at::Tensor py_residual_relu_backward(const at::Tensor& y, const at::Tensor& ga, const std::optional<at::Tensor>& gb) {
  check_join_operand(y, y, "residual_relu_backward", "y");
  check_join_operand(y, ga, "residual_relu_backward", "ga");
  if (gb) check_join_operand(y, *gb, "residual_relu_backward", "gb");
  const int dt = cgx_dtype(y);
  c10::cuda::CUDAGuard guard(y.device());
  at::Tensor g = at::empty_like(y);
  cuda_check(launch_residual_relu_backward(y.data_ptr(), ga.data_ptr(), gb ? gb->data_ptr() : nullptr, g.data_ptr(),
                                           dt, (uint64_t)y.numel(), c10::cuda::getCurrentCUDAStream()),
             "residual_relu_backward");
  return g;
}

// [len(layers), len(candidates)] float64: squared quantization error of every layer at every
// candidate width (common/quant_error.h); CPU tensors run the C++ path, CUDA tensors the kernel
at::Tensor py_quantization_error(const at::Tensor& t, const std::vector<LayerTuple>& layers,
                                 const std::vector<int64_t>& candidates, bool stochastic, double prescale,
                                 bool skip_incomplete) {
  TORCH_CHECK(t.device().is_cpu() || t.is_cuda(), "quantization_error: tensor must be on the CPU or a CUDA device");
  TORCH_CHECK(t.is_contiguous(), "quantization_error: tensor must be contiguous");
  const int dt = cgx_dtype(t);
  const int K = (int)candidates.size();
  TORCH_CHECK(K >= 1 && K <= kQErrMaxCandidates, "quantization_error: need 1 to ", kQErrMaxCandidates,
              " candidate widths, got ", K);
  int bits[kQErrMaxCandidates];
  for (int k = 0; k < K; ++k) {
    TORCH_CHECK(candidates[k] >= 1 && candidates[k] <= 8, "quantization_error: candidate width ", candidates[k],
                " is outside 1..8");
    bits[k] = (int)candidates[k];
  }
  std::vector<QErrLayer> ls;
  ls.reserve(layers.size());
  for (const auto& l : layers) {
    const int64_t off = std::get<0>(l), n = std::get<1>(l), bucket = std::get<3>(l);
    TORCH_CHECK(off >= 0 && n >= 0 && off + n <= t.numel(), "quantization_error: layer (", off, ", ", n,
                ") is outside the tensor of ", t.numel(), " elements");
    TORCH_CHECK(bucket >= 1, "quantization_error: bucket size must be >= 1, got ", bucket);
    // clamped like the plan clamps it (plan.cc: push_segment)
    const uint32_t B = (uint32_t)std::min<int64_t>(bucket, kMaxBlockElems);
    // with skip_incomplete the tail bucket travels raw: no error
    ls.push_back({(uint64_t)off, skip_incomplete ? (uint64_t)n / B * B : (uint64_t)n, B, 0});
  }
  const int64_t L = (int64_t)ls.size();
  if (t.device().is_cpu()) {
    at::Tensor out = at::zeros({L, (int64_t)K}, at::kDouble);
    cpu::quantization_error(t.data_ptr(), dt, ls, bits, K, stochastic, (float)prescale, out.data_ptr<double>());
    return out;
  }
  c10::cuda::CUDAGuard g(t.device());
  auto stream = c10::cuda::getCurrentCUDAStream();
  const std::vector<uint64_t> first = qerr_first(ls);
  const uint64_t nb = first.back();
  TORCH_CHECK(nb < (1ull << 34), "quantization_error: too many buckets for one launch");
  const size_t lbytes = ls.size() * sizeof(QErrLayer), fbytes = first.size() * sizeof(uint64_t);
  // layer table and first buckets go up in one copy from pinned memory: no synchronisation with the stream
  at::Tensor host = at::empty({(int64_t)(lbytes + fbytes)}, at::TensorOptions().dtype(at::kByte).pinned_memory(true));
  std::memcpy(host.data_ptr<uint8_t>(), ls.data(), lbytes);
  std::memcpy(host.data_ptr<uint8_t>() + lbytes, first.data(), fbytes);
  at::Tensor dev = at::empty({(int64_t)(lbytes + fbytes)}, t.options().dtype(at::kByte));
  dev.copy_(host, /*non_blocking=*/true);
  at::Tensor partial = at::empty({(int64_t)std::max<uint64_t>(1, nb * (uint64_t)K)}, t.options().dtype(at::kFloat));
  at::Tensor out = at::empty({L, (int64_t)K}, t.options().dtype(at::kDouble));
  QErrArgs a;
  a.data = t.data_ptr();
  a.dtype = dt;
  a.layer_table = reinterpret_cast<const QErrLayer*>(dev.data_ptr<uint8_t>());
  a.first = reinterpret_cast<const uint64_t*>(dev.data_ptr<uint8_t>() + lbytes);
  a.nbuckets = nb;
  a.layers = (int)L;
  a.bits = bits;
  a.K = K;
  a.prescale = (float)prescale;
  a.stochastic = stochastic;
  a.partial = partial.data_ptr<float>();
  a.out = out.data_ptr<double>();
  cuda_check(launch_quantization_error(a, stream), "quantization_error");
  return out;
}

// ---- training BatchNorm on channels_last input ----
void check_bn_param(const at::Tensor& x, const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.device() == x.device(), "batchnorm_cl: ", name, " must be on ", x.device(),
              ", got ", t.device());
  TORCH_CHECK(t.scalar_type() == at::kFloat, "batchnorm_cl: ", name, " must be float32, got ", t.scalar_type());
  TORCH_CHECK(t.dim() == 1 && t.size(0) == x.size(1) && t.is_contiguous(), "batchnorm_cl: ", name,
              " must be a contiguous vector of ", x.size(1), " channels, got sizes ", t.sizes());
}

// The arrival counters of the chain kernels reset themselves, so one zeroed buffer per device and stream
// serves every launch on that stream. Under CUDA graph capture a zeroing memset would be recorded, not
// run, so a captured call gets its own zeroed counters, allocated (and zeroed) inside the graph.
int* bn_semaphores(const at::Tensor& x, int need, at::Tensor& per_call) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, at::Tensor> cache;
  const auto stream = c10::cuda::getCurrentCUDAStream();
  cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
  cuda_check(cudaStreamIsCapturing(stream.stream(), &capture), "cudaStreamIsCapturing");
  if (capture != cudaStreamCaptureStatusNone) {
    per_call = at::zeros({need}, x.options().dtype(at::kInt));
    return per_call.data_ptr<int>();
  }
  std::lock_guard<std::mutex> lock(mu);
  at::Tensor& t = cache[{(int)x.get_device(), stream.stream()}];
  if (!t.defined() || t.numel() < need) t = at::zeros({need}, x.options().dtype(at::kInt));
  return t.data_ptr<int>();
}

void check_bn_input(const at::Tensor& x, const char* op, const char* name) {
  TORCH_CHECK(x.is_cuda(), op, ": ", name, " must be a CUDA tensor, got ", x.device());
  TORCH_CHECK(x.dim() == 4, op, ": ", name, " must be 4-D, got sizes ", x.sizes());
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast), op, ": ", name,
              " must be channels_last, got strides ", x.strides());
  TORCH_CHECK(x.numel() > 0 && x.numel() <= std::numeric_limits<int32_t>::max(), op, ": ", name,
              " must have 1 to 2^31 - 1 elements, got ", x.numel());
}

std::tuple<at::Tensor, at::Tensor, at::Tensor> py_batchnorm_cl_backward(const at::Tensor& g, const at::Tensor& x,
                                                                        const at::Tensor& weight,
                                                                        const at::Tensor& bias,
                                                                        const at::Tensor& mean,
                                                                        const at::Tensor& invstd, bool relu) {
  check_bn_input(x, "batchnorm_cl_backward", "x");
  check_join_operand(x, g, "batchnorm_cl_backward", "g");
  check_bn_param(x, weight, "weight");
  check_bn_param(x, bias, "bias");
  check_bn_param(x, mean, "mean");
  check_bn_param(x, invstd, "invstd");
  c10::cuda::CUDAGuard guard(x.device());
  BnBackwardArgs a{};
  a.dtype = cgx_dtype(x);
  a.C = (int)x.size(1);
  a.M = (int)(x.numel() / a.C);
  const auto fopt = x.options().dtype(at::kFloat);
  at::Tensor gx = at::empty_like(x);
  at::Tensor sums = at::empty({2, a.C}, fopt);
  at::Tensor gw = at::empty({a.C}, fopt), gb = at::empty({a.C}, fopt);
  at::Tensor staging, sem_call;
  const int gy = batchnorm_cl_grid_y(a.M, a.C);
  if (gy > 1) {
    staging = at::empty({2 * (int64_t)gy * a.C}, fopt);
    a.staging = staging.data_ptr<float>();
  }
  a.sem_len = a.C / 4 + 1;
  a.sem = bn_semaphores(x, a.sem_len, sem_call);
  a.g = g.data_ptr();
  a.x = x.data_ptr();
  a.gx = gx.data_ptr();
  a.weight = weight.data_ptr<float>();
  a.bias = bias.data_ptr<float>();
  a.mean = mean.data_ptr<float>();
  a.invstd = invstd.data_ptr<float>();
  a.sum_dy = sums.data_ptr<float>();
  a.sum_dy_xmu = a.sum_dy + a.C;
  a.grad_weight = gw.data_ptr<float>();
  a.grad_bias = gb.data_ptr<float>();
  a.relu = relu;
  cuda_check(launch_batchnorm_cl_backward(a, c10::cuda::getCurrentCUDAStream()), "batchnorm_cl_backward");
  return {gx, gw, gb};
}

std::tuple<at::Tensor, at::Tensor, at::Tensor> py_batchnorm_cl_forward(const at::Tensor& x, const at::Tensor& weight,
                                                                       const at::Tensor& bias,
                                                                       const at::Tensor& running_mean,
                                                                       const at::Tensor& running_var, double momentum,
                                                                       double eps, bool relu) {
  check_bn_input(x, "batchnorm_cl_forward", "x");
  check_bn_param(x, weight, "weight");
  check_bn_param(x, bias, "bias");
  check_bn_param(x, running_mean, "running_mean");
  check_bn_param(x, running_var, "running_var");
  c10::cuda::CUDAGuard guard(x.device());
  BnForwardArgs a{};
  a.dtype = cgx_dtype(x);
  a.C = (int)x.size(1);
  a.M = (int)(x.numel() / a.C);
  at::Tensor y = at::empty_like(x);
  at::Tensor mean = at::empty({a.C}, x.options().dtype(at::kFloat));
  at::Tensor invstd = at::empty({a.C}, x.options().dtype(at::kFloat));
  at::Tensor staging, sem_call;
  const int gy = batchnorm_cl_grid_y(a.M, a.C);
  if (gy > 1) {
    staging = at::empty({3 * (int64_t)gy * a.C}, x.options().dtype(at::kFloat));
    a.staging = staging.data_ptr<float>();
  }
  a.sem_len = a.C / 4 + 1;
  a.sem = bn_semaphores(x, a.sem_len, sem_call);
  a.x = x.data_ptr();
  a.y = y.data_ptr();
  a.weight = weight.data_ptr<float>();
  a.bias = bias.data_ptr<float>();
  a.running_mean = running_mean.data_ptr<float>();
  a.running_var = running_var.data_ptr<float>();
  a.save_mean = mean.data_ptr<float>();
  a.save_invstd = invstd.data_ptr<float>();
  a.momentum = momentum;
  a.eps = eps;
  a.relu = relu;
  cuda_check(launch_batchnorm_cl_forward(a, c10::cuda::getCurrentCUDAStream()), "batchnorm_cl_forward");
  return {y, mean, invstd};
}

c10::intrusive_ptr<c10d::Backend> create_backend(const c10::intrusive_ptr<c10d::Store>& store, int rank, int size,
                                                 const std::chrono::milliseconds& timeout,
                                                 c10::intrusive_ptr<c10d::Backend> cpu_delegate,
                                                 c10::intrusive_ptr<c10d::Backend> cuda_delegate, int local_size,
                                                 c10::intrusive_ptr<c10d::Backend> cpu_local,
                                                 c10::intrusive_ptr<c10d::Backend> cpu_cross,
                                                 c10::intrusive_ptr<c10d::Backend> cuda_local,
                                                 c10::intrusive_ptr<c10d::Backend> cuda_cross) {
  ProcessGroupCGX::Topology topo;
  topo.local_size = local_size;
  topo.cpu_local = std::move(cpu_local);
  topo.cpu_cross = std::move(cpu_cross);
  topo.cuda_local = std::move(cuda_local);
  topo.cuda_cross = std::move(cuda_cross);
  return c10::make_intrusive<ProcessGroupCGX>(store, rank, size, timeout, std::move(cpu_delegate),
                                              std::move(cuda_delegate), std::move(topo));
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "torch_cgx_b200 native core (sm_90a)";
  py::module::import("torch._C._distributed_c10d");

  py::class_<ProcessGroupCGX, c10d::Backend, c10::intrusive_ptr<ProcessGroupCGX>>(m, "ProcessGroupCGX")
      .def("allreduce_bucket", &ProcessGroupCGX::allreduce_bucket, py::arg("tensor"), py::arg("bucket_idx"),
           py::arg("average") = false, py::call_guard<py::gil_scoped_release>())
      .def("reduce_scatter_compressed",
           [](ProcessGroupCGX& pg, at::Tensor out, at::Tensor in, bool average, int bits, int bucket_size,
              bool skip_incomplete, bool stochastic, int64_t seed, bool overlapped,
              const std::vector<LayerTuple>& layers) {
             return pg.sharded_compressed(ShardedOp::kReduceScatter, out, in, average, bits, bucket_size,
                                          skip_incomplete, stochastic, seed, overlapped, to_layers(layers));
           },
           py::arg("output"), py::arg("input"), py::arg("average") = false, py::arg("bits") = 4,
           py::arg("bucket_size") = 512, py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
           py::arg("seed") = -1, py::arg("overlapped") = false, py::arg("layers") = std::vector<LayerTuple>{},
           py::call_guard<py::gil_scoped_release>())
      .def("all_gather_compressed",
           [](ProcessGroupCGX& pg, at::Tensor out, at::Tensor in, int bits, int bucket_size, bool stochastic,
              int64_t seed, bool overlapped, const std::vector<LayerTuple>& layers) {
             return pg.sharded_compressed(ShardedOp::kAllGather, out, in, false, bits, bucket_size, false,
                                          stochastic, seed, overlapped, to_layers(layers));
           },
           py::arg("output"), py::arg("input"), py::arg("bits") = 4, py::arg("bucket_size") = 512,
           py::arg("stochastic") = false, py::arg("seed") = -1, py::arg("overlapped") = false,
           py::arg("layers") = std::vector<LayerTuple>{}, py::call_guard<py::gil_scoped_release>())
      .def("init_cuda", &ProcessGroupCGX::init_cuda, py::call_guard<py::gil_scoped_release>())
      .def("p2p_ready", &ProcessGroupCGX::p2p_ready)
      .def("lanes", &ProcessGroupCGX::lanes)
      .def("local_size", &ProcessGroupCGX::local_size)
      .def("stats", &ProcessGroupCGX::stats)
      .def("reset_stats", &ProcessGroupCGX::reset_stats)
      .def("check_health", &ProcessGroupCGX::check_health)
      .def("failure", &ProcessGroupCGX::failure)
      .def("last_lanes", &ProcessGroupCGX::last_lanes)
      .def("abort", &ProcessGroupCGX::abort, py::call_guard<py::gil_scoped_release>())
      .def("uses_multicast", [](ProcessGroupCGX& pg) { return pg.uses_multicast(); })
      .def("heap_kind", [](ProcessGroupCGX& pg) { return pg.heap_kind(); })
      .def("enable_trace", &ProcessGroupCGX::enable_trace)
      .def("read_trace", &ProcessGroupCGX::read_trace);

  py::class_<HookState, std::shared_ptr<HookState>>(m, "NativeHookState")
      .def_property_readonly("step", [](const HookState& h) { return h.step.load(); })
      .def_readonly("layer_min_size", &HookState::layer_min_size)
      .def_readonly("bits", &HookState::bits)
      .def_readonly("bucket_size", &HookState::bucket_size)
      .def_readonly("register_step", &HookState::register_step);
  m.def("register_native_hook",
        [](const std::shared_ptr<c10d::Reducer>& reducer, const c10::intrusive_ptr<ProcessGroupCGX>& pg,
           int64_t layer_min_size, int bits, int bucket_size, int register_step) {
          return register_native_hook(reducer, pg, layer_min_size, bits, bucket_size, register_step);
        },
        py::arg("reducer"), py::arg("backend"), py::arg("layer_min_size"), py::arg("bits"), py::arg("bucket_size"),
        py::arg("register_step") = 2);

  m.def("create_backend", &create_backend, py::arg("store"), py::arg("rank"), py::arg("size"), py::arg("timeout"),
        py::arg("cpu_delegate"), py::arg("cuda_delegate"), py::arg("local_size") = 0,
        py::arg("cpu_local") = nullptr, py::arg("cpu_cross") = nullptr, py::arg("cuda_local") = nullptr,
        py::arg("cuda_cross") = nullptr, py::call_guard<py::gil_scoped_release>());

  // reference pybind surface
  m.def("register_layer", [](unsigned bucket_idx, unsigned layer_idx, int64_t numel, int bits, int bucket_size) {
    LayerRegistry::instance().register_layer(bucket_idx, layer_idx, numel, bits, bucket_size);
  });
  m.def("set_quantization_bits", [](unsigned bucket_idx, unsigned layer_idx, int bits) {
    LayerRegistry::instance().set_bits(bucket_idx, layer_idx, bits);
  });
  m.def("set_quantization_bucket_size", [](unsigned bucket_idx, unsigned layer_idx, int bucket_size) {
    LayerRegistry::instance().set_bucket_size(bucket_idx, layer_idx, bucket_size);
  });
  m.def("reset_layers", []() { LayerRegistry::instance().reset(); });
  m.def("num_registered_buckets", []() { return (int64_t)LayerRegistry::instance().num_buckets(); });
  m.def("registered_bucket", [](unsigned bucket_idx) {
    std::vector<std::tuple<int64_t, int, int>> out;
    auto sizes = LayerRegistry::instance().bucket_layer_sizes(bucket_idx);
    for (size_t i = 0; i < sizes.size(); ++i) {
      auto c = LayerRegistry::instance().layer_config(bucket_idx, (unsigned)i);
      out.emplace_back(sizes[i], c.bits, c.bucket_size);
    }
    return out;
  });
  m.def("extract_layers", [](int64_t numel, int explicit_bucket) {
    CompressionEnv env = CompressionEnv::read();
    EngineConfig cfg = EngineConfig::read();
    int resolved = -1;
    auto ls = LayerRegistry::instance().extract(numel, env, cfg.min_compress_elems, explicit_bucket, &resolved);
    std::vector<LayerTuple> out;
    for (auto& l : ls) out.emplace_back((int64_t)l.elem_off, (int64_t)l.numel, (int64_t)l.bits, (int64_t)l.bucket);
    return std::make_pair(out, resolved);
  }, py::arg("numel"), py::arg("explicit_bucket") = -1);

  m.def("engine_config", []() {
    EngineConfig c = EngineConfig::read();
    CompressionEnv e = CompressionEnv::read();
    py::dict d;
    d["fusion_bytes"] = c.fusion_bytes;
    d["min_compress_elems"] = c.min_compress_elems;
    d["fake_ratio"] = c.fake_ratio;
    d["inner_comm"] = to_string(c.inner_comm);
    d["cross_comm"] = to_string(c.cross_comm);
    d["inner_reduction"] = to_string(c.inner_reduction);
    d["cross_reduction"] = to_string(c.cross_reduction);
    d["intra_broadcast"] = c.intra_broadcast;
    d["intra_compress"] = c.intra_compress;
    d["dummy_compression"] = c.dummy_compression;
    d["remote_buf"] = c.remote_buf;
    d["oneshot_max_bytes"] = c.oneshot_max_bytes;
    d["lanes"] = c.lanes;
    d["timeout_ms"] = c.timeout_ms;
    d["local_size"] = c.local_size;
    d["bits"] = e.bits;
    d["bucket_size"] = e.bucket_size;
    d["skip_incomplete"] = e.skip_incomplete;
    d["stochastic"] = e.stochastic;
    d["seed"] = e.seed;
    return d;
  });

  m.def("build_plan", [](const std::vector<LayerTuple>& layers, int world, int lanes, int dtype, bool skip_incomplete,
                         int64_t min_lane_elems) {
    return plan_to_dict(build_plan(to_layers(layers), make_opts(world, lanes, dtype, skip_incomplete, min_lane_elems)));
  }, py::arg("layers"), py::arg("world"), py::arg("lanes"), py::arg("dtype") = 0, py::arg("skip_incomplete") = false,
        py::arg("min_lane_elems") = 2048);
  m.def("reduce_scatter_windows", [](const std::vector<LayerTuple>& shard_layers, int world, int lanes, int dtype,
                                     bool skip_incomplete, int64_t min_lane_elems, int64_t slot_bytes) {
    std::vector<std::vector<LayerTuple>> out;
    for (auto& w : reduce_scatter_windows(to_layers(shard_layers),
                                          make_opts(world, lanes, dtype, skip_incomplete, min_lane_elems),
                                          (uint32_t)slot_bytes)) {
      std::vector<LayerTuple> o;
      for (auto& l : w) o.emplace_back((int64_t)l.elem_off, (int64_t)l.numel, (int64_t)l.bits, (int64_t)l.bucket);
      out.push_back(std::move(o));
    }
    return out;
  }, py::arg("shard_layers"), py::arg("world"), py::arg("lanes"), py::arg("dtype") = 0,
        py::arg("skip_incomplete") = false, py::arg("min_lane_elems") = 2048, py::arg("slot_bytes"));
  m.def("split_for_fusion", [](const std::vector<LayerTuple>& layers, int elsize, int64_t fusion_bytes) {
    std::vector<std::vector<LayerTuple>> out;
    for (auto& g : split_for_fusion(to_layers(layers), elsize, fusion_bytes)) {
      std::vector<LayerTuple> o;
      for (auto& l : g) o.emplace_back((int64_t)l.elem_off, (int64_t)l.numel, (int64_t)l.bits, (int64_t)l.bucket);
      out.push_back(std::move(o));
    }
    return out;
  });

  m.def("sra_simulate", &py_sra_simulate, py::arg("tensors"), py::arg("layers"), py::arg("lanes") = 1,
        py::arg("average") = false, py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
        py::arg("seed") = 0, py::arg("seq") = 0, py::arg("min_lane_elems") = 2048);
  m.def("reduce_scatter_simulate", &py_reduce_scatter_simulate, py::arg("inputs"), py::arg("outputs"),
        py::arg("shard_layers"), py::arg("lanes") = 1, py::arg("average") = false, py::arg("skip_incomplete") = false,
        py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0, py::arg("min_lane_elems") = 2048);
  m.def("all_gather_simulate", &py_all_gather_simulate, py::arg("inputs"), py::arg("outputs"),
        py::arg("shard_layers"), py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0);
  m.def("oneshot_simulate", &py_oneshot_simulate, py::arg("tensors"), py::arg("layers"), py::arg("lanes") = 1,
        py::arg("average") = false, py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
        py::arg("seed") = 0, py::arg("seq") = 0, py::arg("min_lane_elems") = 2048);
  m.def("quantize", &py_quantize, py::arg("tensor"), py::arg("layers"), py::arg("world") = 1, py::arg("lanes") = 1,
        py::arg("skip_incomplete") = false, py::arg("prescale") = 1.0f, py::arg("stochastic") = false,
        py::arg("seed") = 0, py::arg("seq") = 0, py::arg("rank") = 0, py::arg("phase") = 0,
        py::arg("min_lane_elems") = 2048);
  m.def("dequantize", &py_dequantize, py::arg("wire"), py::arg("like"), py::arg("layers"), py::arg("world") = 1,
        py::arg("lanes") = 1, py::arg("skip_incomplete") = false, py::arg("min_lane_elems") = 2048);

  m.def("scale_", [](at::Tensor t, double s) {
    TORCH_CHECK(t.is_cuda() && t.is_contiguous(), "scale_: contiguous CUDA tensor");
    c10::cuda::CUDAGuard g(t.device());
    cuda_check(launch_scale_inplace(t.data_ptr(), cgx_dtype(t), (uint64_t)t.numel(), (float)s,
                                    c10::cuda::getCurrentCUDAStream()),
               "scale");
    return t;
  });
  m.def("add", [](const at::Tensor& x, const at::Tensor& y) {
    TORCH_CHECK(x.is_cuda() && y.is_cuda() && x.is_contiguous() && y.is_contiguous() && x.numel() == y.numel() &&
                    x.scalar_type() == y.scalar_type(),
                "add: matching contiguous CUDA tensors");
    c10::cuda::CUDAGuard g(x.device());
    at::Tensor out = at::empty_like(x);
    cuda_check(launch_add(x.data_ptr(), y.data_ptr(), out.data_ptr(), cgx_dtype(x), (uint64_t)x.numel(),
                          c10::cuda::getCurrentCUDAStream()),
               "add");
    return out;
  });
  m.def("convert", [](const at::Tensor& x, at::ScalarType dst) {
    TORCH_CHECK(x.is_cuda() && x.is_contiguous(), "convert: contiguous CUDA tensor");
    c10::cuda::CUDAGuard g(x.device());
    at::Tensor out = at::empty_like(x, x.options().dtype(dst));
    cuda_check(launch_convert(x.data_ptr(), cgx_dtype(x), out.data_ptr(), cgx_dtype(out), (uint64_t)x.numel(),
                              c10::cuda::getCurrentCUDAStream()),
               "convert");
    return out;
  });
  m.def("quantization_error", &py_quantization_error, py::arg("tensor"), py::arg("layers"), py::arg("candidates"),
        py::arg("stochastic") = false, py::arg("prescale") = 1.0, py::arg("skip_incomplete") = false);
  m.def("residual_relu_forward", &py_residual_relu_forward, py::arg("a"), py::arg("b"),
        "y = relu(a + b), bit-identical to the eager add + relu_");
  m.def("residual_relu_backward", &py_residual_relu_backward, py::arg("y"), py::arg("ga"), py::arg("gb") = py::none(),
        "g = (y <= 0) ? 0 : ga + gb (ga alone when gb is None), bit-identical to the eager accumulation + "
        "threshold_backward");
  m.def("batchnorm_cl_forward", &py_batchnorm_cl_forward, py::arg("x"), py::arg("weight"), py::arg("bias"),
        py::arg("running_mean"), py::arg("running_var"), py::arg("momentum"), py::arg("eps"), py::arg("relu"),
        "training BatchNorm of a channels_last x (fp32 / fp16 / bf16) with fp32 parameters: (y, save_mean, "
        "save_invstd), running stats updated in place; y = relu_(bn(x)) with relu. Bit-identical to "
        "aten.native_batch_norm (+ relu_)");
  m.def("batchnorm_cl_backward", &py_batchnorm_cl_backward, py::arg("g"), py::arg("x"), py::arg("weight"),
        py::arg("bias"), py::arg("mean"), py::arg("invstd"), py::arg("relu"),
        "backward of batchnorm_cl_forward for g with x's strides: (grad_input, grad_weight, grad_bias), the ReLU "
        "mask recomputed from x. Bit-identical to threshold_backward + aten.native_batch_norm_backward");
  m.def("max_resident_ctas", [](int dtype) { return sra_max_resident_ctas(dtype); }, py::arg("dtype") = 0);

  py::class_<FdChannel>(m, "FdChannel")
      .def(py::init<const std::string&>(), py::arg("hint"))
      .def("name", &FdChannel::name)
      .def("send", &FdChannel::try_send, py::arg("peer_name"), py::arg("fd"), py::arg("kind"), py::arg("src"))
      .def("recv", [](FdChannel& ch, int timeout_ms) -> py::object {
        FdMessage m;
        bool ok;
        {
          py::gil_scoped_release rel;
          ok = ch.try_recv(&m, timeout_ms);
        }
        if (!ok) return py::none();
        return py::make_tuple(m.fd, m.kind, m.src);
      }, py::arg("timeout_ms"));
  py::class_<PreparedCodec>(m, "PreparedCodec")
      .def(py::init<const std::vector<LayerTuple>&, at::ScalarType, int64_t, bool>(), py::arg("layers"),
           py::arg("dtype"), py::arg("device") = 0, py::arg("skip_incomplete") = false)
      .def("wire_bytes", &PreparedCodec::wire_bytes)
      .def("numel", &PreparedCodec::numel)
      .def("num_items", &PreparedCodec::num_items)
      .def("quantize", &PreparedCodec::quantize, py::arg("x"), py::arg("wire"), py::arg("prescale") = 1.0,
           py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0)
      .def("dequantize", &PreparedCodec::dequantize, py::arg("wire"), py::arg("out"));
  py::class_<LocalSraGroup>(m, "LocalSraGroup")
      .def(py::init<int, int, int64_t, int64_t, int64_t>(), py::arg("world"), py::arg("lanes"),
           py::arg("slot_bytes"), py::arg("timeout_ms") = 5000, py::arg("min_lane_elems") = 2048)
      .def("allreduce", &LocalSraGroup::allreduce, py::arg("tensors"), py::arg("layers"), py::arg("average") = false,
           py::arg("skip_incomplete") = false, py::arg("stochastic") = false, py::arg("seed") = 0,
           py::arg("seq") = 0)
      .def("allreduce_oneshot", &LocalSraGroup::allreduce_oneshot, py::arg("tensors"), py::arg("layers"),
           py::arg("average") = false, py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
           py::arg("seed") = 0, py::arg("seq") = 0)
      .def("reduce_scatter", &LocalSraGroup::reduce_scatter, py::arg("inputs"), py::arg("outputs"),
           py::arg("shard_layers"), py::arg("average") = false, py::arg("skip_incomplete") = false,
           py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0)
      .def("all_gather", &LocalSraGroup::all_gather, py::arg("inputs"), py::arg("outputs"), py::arg("shard_layers"),
           py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0)
      .def("check", &LocalSraGroup::check)
      .def("allreduce_with_absent_rank", &LocalSraGroup::allreduce_with_absent_rank, py::arg("tensors"),
           py::arg("layers"), py::arg("absent"))
      .def("abort_all", &LocalSraGroup::abort_all)
      .def("status", &LocalSraGroup::status)
      .def("clear", &LocalSraGroup::clear)
      .def("lanes_used", &LocalSraGroup::lanes_used);
  py::class_<LocalReducerGroup>(m, "LocalReducerGroup")
      .def(py::init<int, const std::string&, int64_t>(), py::arg("world"), py::arg("kind"),
           py::arg("timeout_ms") = 10000)
      .def("allreduce", &LocalReducerGroup::allreduce, py::arg("tensors"), py::arg("layers"),
           py::arg("average") = false, py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
           py::arg("seed") = 0, py::arg("seq") = 0)
      .def("broadcast_compressed", &LocalReducerGroup::broadcast_compressed, py::arg("tensors"), py::arg("layers"),
           py::arg("root"), py::arg("skip_incomplete") = false, py::arg("stochastic") = false, py::arg("seed") = 0,
           py::arg("seq") = 0)
      .def("bytes_sent", &LocalReducerGroup::bytes_sent)
      .def("set_recording", &LocalReducerGroup::set_recording, py::arg("on"))
      .def("messages", &LocalReducerGroup::messages);

  m.attr("MAX_BLOCK_ELEMS") = (int64_t)kMaxBlockElems;
  m.attr("MAX_PEERS") = (int64_t)kMaxPeers;
  m.attr("RAW_BITS") = (int64_t)kRawBits;
}

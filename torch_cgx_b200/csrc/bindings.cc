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
//  * LocalEngineGroup: W AllreduceEngines wired as the process group wires them, in one process,
//    with a log of the stages each one issues.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <pybind11/chrono.h>
#include <pybind11/numpy.h>
#include <torch/extension.h>

#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <thread>
#include <tuple>
#include <variant>
#include <vector>

#include "comm/fd_channel.h"
#include "comm/loopback_communicator.h"
#include "common/a2a.h"
#include "common/bit_allocation.h"
#include "common/block_ops.h"
#include "common/config.h"
#include "common/layers.h"
#include "common/plan.h"
#include "common/quant_error.h"
#include "common/sra_sim.h"
#include "engine/quant_error_table.h"
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
// `prescale`: the factor every contribution is multiplied by first; none means 1/W when averaging, else 1
float sim_prescale(std::optional<double> prescale, bool average, int W) {
  return prescale ? (float)*prescale : average ? 1.0f / (float)W : 1.0f;
}

WireCodec allreduce_codec(const std::optional<std::variant<int64_t, std::string>>& bits,
                          const std::vector<LayerSpec>& layers, bool stochastic);

void py_sra_simulate(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, int lanes,
                     bool average, bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                     int64_t min_lane_elems, std::optional<double> prescale,
                     const std::optional<std::variant<int64_t, std::string>>& bits) {
  TORCH_CHECK(!tensors.empty(), "need tensors");
  const int W = (int)tensors.size();
  const int dt = cgx_dtype(tensors[0]);
  std::vector<void*> bufs;
  for (auto& t : tensors) {
    TORCH_CHECK(t.device().is_cpu() && t.is_contiguous() && cgx_dtype(t) == dt, "sra_simulate: CPU contiguous tensors of one dtype");
    bufs.push_back(t.data_ptr());
  }
  const auto specs = to_layers(layers);
  const WireCodec codec = allreduce_codec(bits, specs, stochastic);
  Plan plan = build_plan(specs, make_opts(W, lanes, dt, skip_incomplete, min_lane_elems));
  sra_simulate(plan, bufs, sim_prescale(prescale, average, W), make_rng(stochastic, seed, seq), codec);
}

void py_oneshot_simulate(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, int lanes,
                         bool average, bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                         int64_t min_lane_elems, std::optional<double> prescale,
                         const std::optional<std::variant<int64_t, std::string>>& bits) {
  TORCH_CHECK(!tensors.empty(), "need tensors");
  const int W = (int)tensors.size();
  const int dt = cgx_dtype(tensors[0]);
  std::vector<void*> bufs;
  for (auto& t : tensors) {
    TORCH_CHECK(t.device().is_cpu() && t.is_contiguous() && cgx_dtype(t) == dt, "oneshot_simulate: CPU contiguous tensors");
    bufs.push_back(t.data_ptr());
  }
  const auto specs = to_layers(layers);
  const WireCodec codec = allreduce_codec(bits, specs, stochastic);
  Plan plan = build_plan(specs, make_opts(1, lanes, dt, skip_incomplete, min_lane_elems));
  oneshot_simulate(plan, bufs, sim_prescale(prescale, average, W), make_rng(stochastic, seed, seq), codec);
}

// The `bits` of every all-to-all, reduce-scatter and all-gather binding: 1..8 or 32 (max-min levels,
// or raw), or the name of an FP8 wire codec, which travels in 8-bit records. The `_sr` codecs round
// stochastically whatever `stochastic` says; the others round to nearest only. Integers are checked
// where they are used, as before; an unknown name, or a round-to-nearest FP8 codec with stochastic
// rounding, raises ValueError naming `op` before anything runs.
using A2aBitsArg = std::variant<int64_t, std::string>;
struct A2aBits {
  int bits;
  WireCodec codec;
};
A2aBits a2a_bits(const A2aBitsArg& arg, bool stochastic, const char* op = "all_to_all") {
  const std::string* name = std::get_if<std::string>(&arg);
  if (name == nullptr) return {(int)std::get<int64_t>(arg), kMaxMin};
  WireCodec codec;
  if (*name == "e4m3")
    codec = kE4M3;
  else if (*name == "e5m2")
    codec = kE5M2;
  else if (*name == "e4m3_pow2")
    codec = kE4M3Pow2;
  else if (*name == "e5m2_pow2")
    codec = kE5M2Pow2;
  else if (*name == "e4m3_sr")
    codec = kE4M3SR;
  else if (*name == "e5m2_sr")
    codec = kE5M2SR;
  else
    throw py::value_error(std::string("cgx ") + op +
                          ": bits must be 1..8, 32, \"e4m3\", \"e5m2\", \"e4m3_pow2\", \"e5m2_pow2\", \"e4m3_sr\" or "
                          "\"e5m2_sr\", got \"" +
                          *name + "\"");
  if (stochastic && !fp8_sr(codec))
    throw py::value_error(std::string("cgx ") + op + ": bits=\"" + *name +
                          "\" rounds to nearest only; stochastic rounding needs integer bits or an _sr format");
  return {8, codec};
}

// The codec of a sharded binding that takes a layer table: None or an integer `bits` keeps max-min
// (the table gives the widths); an FP8 name selects that codec for the table's 8-bit layers, and
// every layer must then have bits 8 or 32. ValueError otherwise, before anything runs.
WireCodec sharded_codec(const std::optional<A2aBitsArg>& bits, const std::vector<LayerSpec>& layers, bool stochastic,
                        const char* op) {
  if (!bits) return kMaxMin;
  const A2aBits wb = a2a_bits(*bits, stochastic, op);
  if (wb.codec != kMaxMin)
    for (const LayerSpec& l : layers)
      if (l.bits != 8 && l.bits < kRawBits)
        throw py::value_error(std::string("cgx ") + op + ": an FP8 format needs layers of bits 8 or 32, got " +
                              std::to_string(l.bits));
  return wb.codec;
}
// the same for the allreduce bindings that take a layer table
WireCodec allreduce_codec(const std::optional<A2aBitsArg>& bits, const std::vector<LayerSpec>& layers,
                          bool stochastic) {
  return sharded_codec(bits, layers, stochastic, "allreduce");
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
                                int64_t min_lane_elems, std::optional<double> prescale,
                                const std::optional<A2aBitsArg>& bits) {
  const auto shard = to_layers(shard_layers);
  const WireCodec codec = sharded_codec(bits, shard, stochastic, "reduce_scatter");
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
  reduce_scatter_simulate(plan, in, out, S, sim_prescale(prescale, average, W), make_rng(stochastic, seed, seq),
                          codec);
}

// the dtype of an all-to-all output: the inputs', or with codes (output_scales) one byte per element,
// uint8 or the codec's float8
bool a2a_output_dtype_ok(const at::Tensor& t, int dt, WireCodec codes_codec) {
  if (codes_codec == kMaxMin) return cgx_dtype(t) == dt;
  const at::ScalarType s = t.scalar_type();
  return s == at::kByte || s == (fp8_base(codes_codec) == kE4M3 ? at::kFloat8_e4m3fn : at::kFloat8_e5m2);
}

// The codes output of the all-gather bindings: outputs[r] holds W * S code bytes (uint8 or the
// codec's float8) and output_scales[r] one contiguous float32 per bucket of it, on the inputs'
// device. ValueError for a codec or table without codes (codes_bucket). Returns the scale pointers.
std::vector<float*> ag_scales(const std::vector<at::Tensor>& inputs, const std::vector<at::Tensor>& outputs,
                              const std::vector<LayerSpec>& shard, WireCodec codec,
                              const std::vector<at::Tensor>& scales) {
  const uint64_t B = codes_bucket(ShardedOp::kAllGather, shard, codec);
  const uint64_t W = inputs.size(), S = shard_elems(shard);
  TORCH_CHECK(W >= 1 && outputs.size() == W && scales.size() == W,
              "all_gather: one input, one output and one output_scales tensor per rank");
  const int dt = cgx_dtype(inputs[0]);
  std::vector<float*> ptrs;
  for (size_t r = 0; r < W; ++r) {
    const at::Tensor &i = inputs[r], &o = outputs[r], &sc = scales[r];
    TORCH_CHECK(i.is_contiguous() && cgx_dtype(i) == dt && i.device() == inputs[0].device() && (uint64_t)i.numel() == S,
                "all_gather: contiguous inputs of S elements, of one dtype and device");
    TORCH_CHECK(o.is_contiguous() && o.device() == i.device() && a2a_output_dtype_ok(o, dt, codec) &&
                    (uint64_t)o.numel() == W * S,
                "all_gather: rank ", r, "'s codes output must be a contiguous uint8 or ",
                fp8_base(codec) == kE4M3 ? "float8_e4m3fn" : "float8_e5m2", " tensor of W * S elements on the inputs' device");
    TORCH_CHECK(sc.is_contiguous() && sc.device() == i.device() && sc.scalar_type() == at::kFloat &&
                    (uint64_t)sc.numel() * B == W * S,
                "all_gather: rank ", r, "'s output_scales must be a contiguous float32 tensor of one element per ",
                "bucket of its output, on the inputs' device");
    ptrs.push_back(sc.data_ptr<float>());
  }
  return ptrs;
}

// All-gather oracle (ag_kernel): shard q is one quantization round trip (roundtrip_simulate) of
// in_q placed at q * S, through copy q of the replicated table and rank q's publish stream (phase
// 1, the SRA's requantization), so the RNG counters are the kernel's element indices. Every output
// gets the same bytes.
// With `output_scales` (an FP8 `bits`): the codes output, shard q's records of that round trip
// undecoded (codes_simulate) at q * S of every output and q * S / B of every scales tensor.
void py_all_gather_simulate(const std::vector<at::Tensor>& inputs, std::vector<at::Tensor> outputs,
                            const std::vector<LayerTuple>& shard_layers, bool stochastic, uint64_t seed,
                            uint32_t seq, const std::optional<A2aBitsArg>& bits,
                            const std::optional<std::vector<at::Tensor>>& output_scales) {
  const auto shard = to_layers(shard_layers);
  const WireCodec codec = sharded_codec(bits, shard, stochastic, "all_gather");
  if (output_scales) {
    const std::vector<float*> scales = ag_scales(inputs, outputs, shard, codec, *output_scales);
    TORCH_CHECK(inputs[0].device().is_cpu(), "all_gather_simulate: CPU tensors");
    const int W = (int)inputs.size();
    const uint64_t S = shard_elems(shard);
    const size_t es = (size_t)dtype_size(cgx_dtype(inputs[0])), per_copy = shard.size();
    const auto layers = replicate(shard, W, S);
    std::vector<uint8_t> full((size_t)W * S * es);  // the shards where the plan addresses them
    for (int q = 0; q < W; ++q) std::memcpy(full.data() + (size_t)q * S * es, inputs[q].data_ptr(), S * es);
    uint8_t* codes0 = static_cast<uint8_t*>(outputs[0].data_ptr());
    for (int q = 0; q < W; ++q) {
      const std::vector<LayerSpec> copy(layers.begin() + (ptrdiff_t)(q * per_copy),
                                        layers.begin() + (ptrdiff_t)((q + 1) * per_copy));
      codes_simulate(build_plan(copy, make_opts(1, 1, cgx_dtype(inputs[0]), false, 1 << 30)), full.data(), codes0,
                     scales[0], codec, make_rng_key(make_rng(stochastic, seed, seq), q, 1));
    }
    for (int r = 1; r < W; ++r) {
      std::memcpy(outputs[r].data_ptr(), codes0, (size_t)W * S);
      std::memcpy(scales[r], scales[0], (size_t)output_scales->at(0).numel() * sizeof(float));
    }
    return;
  }
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
                       make_rng(stochastic, seed, seq), q, 1, codec);
  }
  for (int r = 1; r < W; ++r) std::memcpy(outputs[r].data_ptr(), out0, S * W * es);
}

// ---- all-to-all: counts[q][r] elements go from rank q to rank r ------------------------------
using CountMatrix = std::vector<std::vector<int64_t>>;
// one optional row index per virtual rank (the routed all-to-all)
using IndexList = std::vector<std::optional<at::Tensor>>;

std::vector<std::vector<uint64_t>> check_counts(const CountMatrix& counts, size_t W) {
  TORCH_CHECK(counts.size() == W, "all_to_all: counts must be a W x W matrix");
  std::vector<std::vector<uint64_t>> out(W, std::vector<uint64_t>(W));
  for (size_t q = 0; q < W; ++q) {
    TORCH_CHECK(counts[q].size() == W, "all_to_all: counts must be a W x W matrix");
    for (size_t r = 0; r < W; ++r) {
      TORCH_CHECK(counts[q][r] >= 0, "all_to_all: negative count");
      out[q][r] = (uint64_t)counts[q][r];
    }
  }
  return out;
}

// The codes output of the all-to-all bindings: `output_scales` holds one contiguous float32 tensor
// per rank, on the side of the outputs, with one element per bucket of the rank's output; the
// outputs then hold codes (a2a_output_dtype_ok). Returns the pointers (empty: decoded output).
std::vector<float*> a2a_scales(const std::optional<std::vector<at::Tensor>>& scales,
                               const std::vector<at::Tensor>& outputs, const A2aBits& wb, int64_t bucket) {
  std::vector<float*> ptrs;
  if (!scales) return ptrs;
  if (wb.codec == kMaxMin) throw py::value_error("cgx all_to_all: output_scales needs bits \"e4m3\" or \"e5m2\"");
  if (bucket < 1 || bucket > (int64_t)kMaxBlockElems)
    throw py::value_error("cgx all_to_all: output_scales needs 1 <= bucket_size <= " + std::to_string(kMaxBlockElems));
  TORCH_CHECK(scales->size() == outputs.size(), "all_to_all: one output_scales tensor per rank");
  for (size_t r = 0; r < outputs.size(); ++r) {
    const at::Tensor& s = (*scales)[r];
    TORCH_CHECK(s.scalar_type() == at::kFloat && s.is_contiguous() && s.is_cuda() == outputs[r].is_cuda() &&
                    s.numel() * bucket == outputs[r].numel(),
                "all_to_all: rank ", r, "'s output_scales must be a contiguous float32 tensor of one element per ",
                "bucket of its output, on the outputs' device");
    ptrs.push_back(s.data_ptr<float>());
  }
  return ptrs;
}

// rank r's input holds row r of the matrix, its output column r
void check_a2a_tensors(const std::vector<at::Tensor>& inputs, const std::vector<at::Tensor>& outputs,
                       const std::vector<std::vector<uint64_t>>& counts, bool cuda, WireCodec codes_codec = kMaxMin) {
  const size_t W = counts.size();
  TORCH_CHECK(inputs.size() == W && outputs.size() == W, "all_to_all: one input and one output per rank");
  const int dt = cgx_dtype(inputs[0]);
  for (size_t r = 0; r < W; ++r) {
    uint64_t nin = 0, nout = 0;
    for (size_t q = 0; q < W; ++q) {
      nin += counts[r][q];
      nout += counts[q][r];
    }
    for (const at::Tensor* t : {&inputs[r], &outputs[r]})
      TORCH_CHECK(t->is_cuda() == cuda && t->is_contiguous() &&
                      (t == &inputs[r] ? cgx_dtype(*t) == dt : a2a_output_dtype_ok(*t, dt, codes_codec)),
                  "all_to_all: contiguous tensors of one dtype, all on ", cuda ? "the GPU" : "the CPU");
    TORCH_CHECK((uint64_t)inputs[r].numel() == nin && (uint64_t)outputs[r].numel() == nout,
                "all_to_all: rank ", r, "'s tensors do not match its row and column of the counts");
  }
}

void py_all_to_all_simulate(const std::vector<at::Tensor>& inputs, std::vector<at::Tensor> outputs,
                            const CountMatrix& counts_in, const A2aBitsArg& bits_arg, int64_t bucket, bool stochastic,
                            uint64_t seed, uint32_t seq, const std::optional<std::vector<at::Tensor>>& output_scales) {
  const A2aBits wb = a2a_bits(bits_arg, stochastic);
  const auto counts = check_counts(counts_in, inputs.size());
  const std::vector<float*> scales = a2a_scales(output_scales, outputs, wb, bucket);
  check_a2a_tensors(inputs, outputs, counts, false, output_scales ? wb.codec : kMaxMin);
  std::vector<const void*> in;
  std::vector<void*> out;
  for (size_t r = 0; r < inputs.size(); ++r) {
    in.push_back(inputs[r].data_ptr());
    out.push_back(outputs[r].data_ptr());
  }
  all_to_all_simulate(cgx_dtype(inputs[0]), in, out, counts, wb.bits, wb.codec, (uint32_t)bucket,
                      make_rng(stochastic, seed, seq), output_scales ? &scales : nullptr);
}

// The cross-node all-to-all's buffers for world rank `rank` with nodes of `local_size` ranks
// (a2a_remote_params): counts[q] elements for or from rank q; returns (record bytes per rank,
// region offset per rank, buffer bytes).
// a2a_remote_params after checking its arguments; returns the buffer's bytes
int64_t remote_params(A2aRemoteParams& p, const std::vector<int64_t>& counts, int rank, int local_size,
                      const A2aBits& wb, int64_t bucket, int dtype, const char* what,
                      std::vector<uint64_t>* wire = nullptr, std::vector<uint64_t>* region = nullptr) {
  TORCH_CHECK(local_size >= 1 && !counts.empty() && (int64_t)counts.size() <= kA2aMaxWorld &&
                  counts.size() % (size_t)local_size == 0 && rank >= 0 && rank < (int)counts.size(),
              what, ": 1..", kA2aMaxWorld, " counts, a multiple of local_size, and a rank among them");
  TORCH_CHECK(bucket >= 1, what, ": bucket_size must be >= 1");
  for (int64_t n : counts) TORCH_CHECK(n >= 0 && n < (1ll << 32), what, ": counts must be in [0, 2^32)");
  std::vector<uint64_t> c(counts.begin(), counts.end()), w, r;
  return (int64_t)a2a_remote_params(p, c, rank, local_size, dtype, wb.bits, wb.codec, (uint32_t)bucket,
                                    wire ? wire : &w, region ? region : &r);
}

std::tuple<std::vector<int64_t>, std::vector<int64_t>, int64_t> py_a2a_remote_wire(const std::vector<int64_t>& counts,
                                                                                   int rank, int local_size,
                                                                                   const A2aBitsArg& bits, int64_t bucket,
                                                                                   int dtype) {
  auto p = std::make_unique<A2aRemoteParams>();
  std::vector<uint64_t> wire, region;
  const int64_t total =
      remote_params(*p, counts, rank, local_size, a2a_bits(bits, false), bucket, dtype, "a2a_remote_wire", &wire, &region);
  return {std::vector<int64_t>(wire.begin(), wire.end()), std::vector<int64_t>(region.begin(), region.end()), total};
}

// One launch of the pack (a2a_pack) or unpack kernel on the current stream, as the engine launches
// it for world rank `rank` (a2a_remote_params): pack quantizes every chunk of `input` for a rank of
// another node into the returned buffer (or `out`); unpack decodes `records` (such a buffer) into
// those chunks' rows of `output`, or with output_scales unpacks their codes and units.
at::Tensor py_a2a_pack(const at::Tensor& input, const std::vector<int64_t>& counts, int rank, int local_size,
                       const A2aBitsArg& bits, int64_t bucket, bool stochastic, uint64_t seed, uint32_t seq,
                       const std::optional<at::Tensor>& out) {
  const A2aBits wb = a2a_bits(bits, stochastic);
  TORCH_CHECK(input.is_cuda() && input.is_contiguous(), "a2a_pack: a contiguous CUDA input");
  TORCH_CHECK(wb.bits < kRawBits, "a2a_pack: raw chunks travel as their bytes, nothing is packed");
  const int dt = cgx_dtype(input);
  int64_t n = 0;
  for (int64_t c : counts) n += c;
  TORCH_CHECK(input.numel() == n, "a2a_pack: the input holds ", input.numel(), " elements, the counts ", n);
  auto p = std::make_unique<A2aRemoteParams>();
  const int64_t total = remote_params(*p, counts, rank, local_size, wb, bucket, dt, "a2a_pack");
  at::Tensor buf = out ? *out : at::zeros({total + 16}, input.options().dtype(at::kByte));
  TORCH_CHECK(buf.is_cuda() && buf.is_contiguous() && buf.scalar_type() == at::kByte && buf.numel() >= total,
              "a2a_pack: out must be a contiguous CUDA uint8 tensor of at least ", total, " bytes");
  c10::cuda::CUDAGuard g(input.device());
  p->in = input.data_ptr();
  p->out = buf.data_ptr();
  p->rng = make_rng_key(make_rng(stochastic, seed, seq), rank, 0);
  cuda_check(launch_a2a_pack(*p, c10::cuda::getCurrentCUDAStream().stream()), "launch_a2a_pack");
  return buf;
}

void py_a2a_unpack(const at::Tensor& records, at::Tensor output, const std::vector<int64_t>& counts, int rank,
                   int local_size, const A2aBitsArg& bits, int64_t bucket, const std::optional<at::Tensor>& output_scales) {
  const A2aBits wb = a2a_bits(bits, false);
  TORCH_CHECK(wb.bits < kRawBits, "a2a_unpack: raw chunks travel as their bytes, nothing is unpacked");
  TORCH_CHECK(records.is_cuda() && records.is_contiguous() && records.scalar_type() == at::kByte,
              "a2a_unpack: records must be a contiguous CUDA uint8 tensor");
  TORCH_CHECK(output.is_cuda() && output.is_contiguous(), "a2a_unpack: a contiguous CUDA output");
  const bool codes = output_scales.has_value();
  TORCH_CHECK(!codes || (wb.codec != kMaxMin && output_scales->is_cuda() && output_scales->is_contiguous() &&
                         output_scales->scalar_type() == at::kFloat),
              "a2a_unpack: output_scales needs an FP8 bits and a contiguous CUDA float32 tensor");
  // a codes output has no element type of the sender's: any dtype gives the same records, since the
  // record bytes of compressed (8-bit) blocks do not depend on the element size (block_wire_bytes)
  const int dt = codes ? kF32 : cgx_dtype(output);
  auto p = std::make_unique<A2aRemoteParams>();
  const int64_t total = remote_params(*p, counts, rank, local_size, wb, bucket, dt, "a2a_unpack");
  int64_t n = 0;
  for (int64_t x : counts) n += x;
  TORCH_CHECK(output.numel() == n, "a2a_unpack: the output holds ", output.numel(), " elements, the counts ", n);
  TORCH_CHECK(records.numel() >= total, "a2a_unpack: records hold ", records.numel(), " bytes, need ", total);
  c10::cuda::CUDAGuard g(output.device());
  p->in = records.data_ptr();
  p->out = output.data_ptr();
  p->out_scales = codes ? output_scales->data_ptr<float>() : nullptr;
  cuda_check(launch_a2a_unpack(*p, c10::cuda::getCurrentCUDAStream().stream()), "launch_a2a_unpack");
}

// the items of one chunk from common/a2a.h, rows as in plan_to_dict, offsets in the contiguous image
at::Tensor py_a2a_items(int64_t n, int bits, int64_t bucket, int dtype) {
  const A2aGeom g = a2a_geom((uint32_t)n, bits, (uint32_t)bucket, dtype_size(dtype));
  std::vector<WarpItem> its;
  for (uint32_t b = 0; b < a2a_num_blocks(g); ++b)
    for (uint32_t j = 0; j < a2a_block_num_items(g, a2a_block_n(g, b)); ++j) {
      WarpItem it = a2a_block_item(g, b, j);
      it.meta_off += b * g.block_wire;
      it.pay_off += b * g.block_wire;
      its.push_back(it);
    }
  auto items = at::empty({(int64_t)its.size(), 7}, at::kLong);
  auto* ip = items.data_ptr<int64_t>();
  for (size_t i = 0; i < its.size(); ++i) {
    ip[i * 7 + 0] = its[i].elem_off;
    ip[i * 7 + 1] = its[i].meta_off;
    ip[i * 7 + 2] = its[i].pay_off;
    ip[i * 7 + 3] = item_kind(its[i]);
    ip[i * 7 + 4] = item_lpb_log2(its[i]);
    ip[i * 7 + 5] = item_bits(its[i]);
    ip[i * 7 + 6] = item_n(its[i]);
  }
  return items;
}

// The windows of one chunk: for every lane, a list of windows, each a list of its blocks as
// (first element, elements, wire bytes); plus the lane's share of a slot.
py::dict py_a2a_windows(int64_t n, int bits, int64_t bucket, int dtype, int64_t slot_bytes, int lanes) {
  TORCH_CHECK(lanes >= 1, "a2a_windows: lanes must be >= 1");
  const A2aGeom g = a2a_geom((uint32_t)n, bits, (uint32_t)bucket, dtype_size(dtype));
  const uint32_t share = a2a_lane_slot_bytes((uint32_t)slot_bytes, lanes);
  const uint32_t bpw = a2a_window_blocks(g, share);
  py::dict d;
  d["lane_slot"] = share;
  d["window_blocks"] = bpw;
  d["block_elems"] = g.block_elems;
  d["block_wire"] = g.block_wire;
  std::vector<std::vector<std::vector<std::tuple<int64_t, int64_t, int64_t>>>> lanes_out(lanes);
  if (bpw > 0) {
    for (int c = 0; c < lanes; ++c) {
      const uint32_t nw = a2a_lane_windows(g, c, lanes, bpw);
      const uint32_t lb = a2a_lane_blocks(a2a_num_blocks(g), c, lanes);
      for (uint32_t k = 0; k < nw; ++k) {
        std::vector<std::tuple<int64_t, int64_t, int64_t>> w;
        for (uint32_t j = k * bpw; j < lb && j < (k + 1) * bpw; ++j) {
          const uint32_t b = (uint32_t)c + j * (uint32_t)lanes, bn = a2a_block_n(g, b);
          w.emplace_back((int64_t)b * g.block_elems, (int64_t)bn, (int64_t)block_wire_bytes(bn, g.bits, g.bucket, g.elsize));
        }
        lanes_out[c].push_back(std::move(w));
      }
    }
  }
  d["lanes"] = lanes_out;
  return d;
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
    c10::cuda::CUDAGuard g((c10::DeviceIndex)device);
    cudaStream_t s = c10::cuda::getCurrentCUDAStream().stream();
    dp_ = &plans_.get(to_layers(layers), make_opts(1, 1, cgx_dtype(probe), skip_incomplete, 1 << 30), s);
    plans_.upload(*dp_, s);
    cuda_check(cudaStreamSynchronize(s), "upload items");  // the calls may run on any stream
  }
  int64_t wire_bytes() const { return (int64_t)wire_row_bytes(dp_->plan); }
  int64_t numel() const { return (int64_t)dp_->plan.numel; }
  int64_t num_items() const { return (int64_t)dp_->plan.items.size(); }
  void quantize(const at::Tensor& x, at::Tensor& wire, double prescale, bool stochastic, uint64_t seed, uint32_t seq) {
    check(x, wire);
    c10::cuda::CUDAGuard g(x.device());
    ops_->quantize(*dp_, x.data_ptr(), 0, (uint32_t)dp_->plan.blocks.size(), wire.data_ptr<uint8_t>(), (float)prescale,
                   make_rng_key(make_rng(stochastic, seed, seq), 0, 0), c10::cuda::getCurrentCUDAStream());
  }
  void dequantize(const at::Tensor& wire, at::Tensor& out) {
    check(out, wire);
    c10::cuda::CUDAGuard g(out.device());
    ops_->dequantize(*dp_, wire.data_ptr<uint8_t>(), 0, (uint32_t)dp_->plan.blocks.size(), out.data_ptr(),
                     c10::cuda::getCurrentCUDAStream());
  }

 private:
  void check(const at::Tensor& x, const at::Tensor& wire) const {
    TORCH_CHECK(x.is_cuda() && x.is_contiguous() && cgx_dtype(x) == dp_->plan.dtype &&
                    (uint64_t)x.numel() == dp_->plan.numel,
                "PreparedCodec: tensor does not match the prepared layout");
    TORCH_CHECK(wire.is_cuda() && wire.is_contiguous() && wire.scalar_type() == at::kByte &&
                    (size_t)wire.numel() >= wire_row_bytes(dp_->plan),
                "PreparedCodec: wire buffer too small");
  }
  PlanCache plans_{1};
  const DevicePlan* dp_ = nullptr;
  std::unique_ptr<BlockBackend> ops_ = make_cuda_block_backend();
};

// ---- single-process multi-rank harness --------------------------------------
// The combine arguments of the virtual-rank all-to-all bindings: gate[r] (CUDA float32 [T, k],
// k <= 32) and combine_out[r] (T * row elements of the inputs' dtype) for every rank r that
// combines; ValueError on malformed ones. Fills routes[r]'s combine fields (topk 0: no combine)
// and returns the zeroed arrival masks of the fused kernel, to be kept until the call returns.
std::vector<at::Tensor> combine_routes(std::vector<A2aRoute>& routes, const std::vector<at::Tensor>& inputs,
                                       const IndexList& gate, const IndexList& combine_out, const A2aBits& wb,
                                       int64_t bucket, int64_t row, bool codes) {
  std::vector<at::Tensor> masks;
  if (gate.empty() && combine_out.empty()) return masks;
  TORCH_CHECK_VALUE(gate.size() == routes.size() && combine_out.size() == routes.size(),
                    "all_to_all: one gate and one combine_out per rank");
  TORCH_CHECK_VALUE(!codes, "cgx all_to_all: a codes output (output_scales) has no combine");
  for (size_t r = 0; r < routes.size(); ++r) {
    TORCH_CHECK_VALUE(gate[r].has_value() == combine_out[r].has_value(),
                      "all_to_all: rank ", r, " needs both a gate and a combine_out, or neither");
    if (!gate[r]) continue;
    const at::Tensor &g = *gate[r], &o = *combine_out[r];
    TORCH_CHECK_VALUE(g.is_cuda() && g.scalar_type() == at::kFloat && g.is_contiguous() && g.dim() == 2,
                      "all_to_all: rank ", r, "'s gate must be a contiguous CUDA float32 tensor [T, k]");
    const int64_t T = g.size(0), k = g.size(1);
    TORCH_CHECK_VALUE(k >= 1 && k <= 32, "all_to_all: rank ", r, "'s gate has k = ", k, ", not in 1..32");
    A2aRoute& rt = routes[r];
    TORCH_CHECK_VALUE(rt.out_index != nullptr && rt.out_rows == (uint64_t)(T * k), "all_to_all: rank ", r,
                      " combines through an output_index into T * k = ", T * k, " slots");
    TORCH_CHECK_VALUE(o.is_cuda() && o.is_contiguous() && o.scalar_type() == inputs[r].scalar_type() &&
                          o.numel() == T * row,
                      "all_to_all: rank ", r, "'s combine_out must be T * row contiguous elements of the inputs' dtype");
    rt.combine_out = o.data_ptr();
    rt.gate = g.data_ptr<float>();
    rt.topk = (uint32_t)k;
    const int64_t span = a2a_row_span(wb.bits, (uint32_t)bucket, dtype_size(cgx_dtype(inputs[r])));
    masks.push_back(at::zeros({T * (row / span)}, g.options().dtype(at::kInt)));
    rt.masks = reinterpret_cast<uint32_t*>(masks.back().data_ptr<int32_t>());
  }
  return masks;
}

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
  // `bits`: None or an integer keeps max-min, an FP8 format name sends the 8-bit layers as FP8
  void allreduce_oneshot(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, bool average,
                         bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                         const std::optional<A2aBitsArg>& bits) {
    run(std::move(tensors), layers, average, skip_incomplete, stochastic, seed, seq, true, -1,
        allreduce_codec(bits, to_layers(layers), stochastic));
  }
  void allreduce(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, bool average,
                 bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                 const std::optional<A2aBitsArg>& bits) {
    run(std::move(tensors), layers, average, skip_incomplete, stochastic, seed, seq, false, -1,
        allreduce_codec(bits, to_layers(layers), stochastic));
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
           bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq, bool oneshot, int absent = -1,
           WireCodec codec = kMaxMin) {
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
            fused_[r]->run_oneshot(*plans[r], tensors[r].data_ptr(), ps, rng, streams_[r].stream(), codec);
          else
            fused_[r]->run(*plans[r], tensors[r].data_ptr(), ps, rng, streams_[r].stream(), codec);
        });
  }

  // reduce-scatter: inputs[r] holds W * S elements of virtual rank r, outputs[r] receives shard r
  // (`bits`: sharded_codec)
  void reduce_scatter(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs,
                      const std::vector<LayerTuple>& shard_layers, bool average, bool skip_incomplete,
                      bool stochastic, uint64_t seed, uint32_t seq, const std::optional<A2aBitsArg>& bits) {
    sharded(ShardedOp::kReduceScatter, inputs, outputs, shard_layers, average, skip_incomplete, stochastic, seed, seq,
            bits);
  }
  // all-gather: inputs[r] holds virtual rank r's shard of S elements, outputs[r] receives W * S
  // (output_scales: the codes output, outputs[r] then one code byte per element, ag_scales)
  void all_gather(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs,
                  const std::vector<LayerTuple>& shard_layers, bool stochastic, uint64_t seed, uint32_t seq,
                  const std::optional<A2aBitsArg>& bits, const std::optional<std::vector<at::Tensor>>& output_scales) {
    sharded(ShardedOp::kAllGather, inputs, outputs, shard_layers, false, false, stochastic, seed, seq, bits,
            output_scales);
  }
  // all-to-all: counts[q][r] elements go from virtual rank q to r; inputs[r] holds row r of the
  // matrix in destination order, outputs[r] receives column r in source order.
  // Routed form (the fused kernel's, so a2a_rows_fit(row, ...) must hold): input_index[r] /
  // output_index[r], when given and not None, are rank r's int64 row indices into inputs[r] /
  // outputs[r], rows of `row` elements; the counts then describe the logical buffers of whole rows.
  // Combine (A2aRoute::combine_out): with gate[r] (CUDA float32 [T, k]) and combine_out[r] ([T, row]
  // elements of the inputs' dtype) outputs[r] is rank r's slots buffer of T * k rows, named by its
  // output_index, and the kernel writes the weighted combine of the slots into combine_out[r].
  // Scaled send (A2aRoute::in_scale): input_scale[r], when given and not None, is a contiguous CUDA
  // float32 vector of one entry per input_index[r] entry; sent row i is T(x * input_scale[r][i]).
  void all_to_all(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs, const CountMatrix& counts_in,
                  const A2aBitsArg& bits_arg, int64_t bucket, bool stochastic, uint64_t seed, uint32_t seq,
                  const IndexList& input_index, const IndexList& output_index, int64_t row,
                  const std::optional<std::vector<at::Tensor>>& output_scales, const IndexList& gate,
                  const IndexList& combine_out, const IndexList& input_scale) {
    const A2aBits wb = a2a_bits(bits_arg, stochastic);
    const auto counts = check_counts(counts_in, (size_t)world_);
    TORCH_CHECK((int)outputs.size() == world_, "all_to_all: one input and one output per rank");
    const std::vector<float*> scales = a2a_scales(output_scales, outputs, wb, bucket);
    const WireCodec codes_codec = output_scales ? wb.codec : kMaxMin;
    const bool routed = !input_index.empty() || !output_index.empty();
    TORCH_CHECK(input_index.empty() || (int)input_index.size() == world_, "all_to_all: one input_index per rank");
    TORCH_CHECK(output_index.empty() || (int)output_index.size() == world_, "all_to_all: one output_index per rank");
    std::vector<A2aRoute> routes((size_t)world_);
    if (routed) {
      TORCH_CHECK(row >= 1, "all_to_all: row must be >= 1");
      for (int r = 0; r < world_; ++r) {
        A2aRoute& rt = routes[r];
        rt.row = (uint64_t)row;
        rt.in_rows = (uint64_t)inputs[r].numel() / (uint64_t)row;
        rt.out_rows = (uint64_t)outputs[r].numel() / (uint64_t)row;
        uint64_t nin = 0, nout = 0;
        for (int q = 0; q < world_; ++q) {
          nin += counts[r][q];
          nout += counts[q][r];
        }
        for (int side = 0; side < 2; ++side) {
          const IndexList& list = side ? output_index : input_index;
          if (list.empty() || !list[r].has_value()) continue;
          const at::Tensor& ix = *list[r];
          TORCH_CHECK(ix.is_cuda() && ix.scalar_type() == at::kLong && ix.dim() == 1 && ix.is_contiguous() &&
                          (uint64_t)ix.numel() * (uint64_t)row == (side ? nout : nin),
                      "all_to_all: rank ", r, "'s ", side ? "output" : "input",
                      "_index must be a contiguous CUDA int64 vector of one entry per row of its counts");
          (side ? rt.out_index : rt.in_index) = ix.data_ptr<int64_t>();
        }
      }
    }
    TORCH_CHECK_VALUE(input_scale.empty() || (int)input_scale.size() == world_, "all_to_all: one input_scale per rank");
    for (int r = 0; r < (int)input_scale.size(); ++r) {
      if (!input_scale[r]) continue;
      const at::Tensor& sc = *input_scale[r];
      TORCH_CHECK_VALUE(routes[r].in_index != nullptr, "all_to_all: rank ", r, "'s input_scale needs an input_index");
      TORCH_CHECK_VALUE(sc.is_cuda() && sc.scalar_type() == at::kFloat && sc.dim() == 1 && sc.is_contiguous() &&
                            sc.numel() == input_index[r]->numel(),
                        "all_to_all: rank ", r, "'s input_scale must be a contiguous CUDA float32 vector of one ",
                        "entry per input_index entry");
      routes[r].in_scale = sc.data_ptr<float>();
    }
    const std::vector<at::Tensor> masks =
        combine_routes(routes, inputs, gate, combine_out, wb, bucket, row, output_scales.has_value());
    for (int r = 0; r < world_; ++r) {
      const bool in_ix = routes[r].in_index != nullptr, out_ix = routes[r].out_index != nullptr;
      uint64_t nin = 0, nout = 0;
      for (int q = 0; q < world_; ++q) {
        nin += counts[r][q];
        nout += counts[q][r];
      }
      for (const at::Tensor* t : {&inputs[r], &outputs[r]})
        TORCH_CHECK(t->is_cuda() && t->is_contiguous() &&
                        (t == &inputs[r] ? cgx_dtype(*t) == cgx_dtype(inputs[0])
                                         : a2a_output_dtype_ok(*t, cgx_dtype(inputs[0]), codes_codec)),
                    "all_to_all: contiguous tensors of one dtype, all on the GPU");
      TORCH_CHECK((in_ix || (uint64_t)inputs[r].numel() == nin) && (out_ix || (uint64_t)outputs[r].numel() == nout),
                  "all_to_all: rank ", r, "'s tensors do not match its row and column of the counts");
    }
    const int dt = cgx_dtype(inputs[0]);
    const RngParams rng = make_rng(stochastic, seed, seq);
    fork_join([](int) {},
              [&](int r) {
                std::vector<uint64_t> out_counts(world_);
                for (int q = 0; q < world_; ++q) out_counts[q] = counts[q][r];
                fused_[r]->all_to_all(inputs[r].data_ptr(), outputs[r].data_ptr(), counts[r], out_counts, dt, wb.bits,
                                      wb.codec, (uint32_t)bucket, rng, streams_[r].stream(), routed ? &routes[r] : nullptr,
                                      scales.empty() ? nullptr : scales[r]);
              });
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
               uint64_t seed, uint32_t seq, const std::optional<A2aBitsArg>& bits,
               const std::optional<std::vector<at::Tensor>>& output_scales = std::nullopt) {
    const bool rs = op == ShardedOp::kReduceScatter;
    const WireCodec codec = sharded_codec(bits, to_layers(shard_layers), stochastic, op_name(op));
    TORCH_CHECK((int)inputs.size() == world_ && (int)outputs.size() == world_,
                "need one input and one output per virtual rank");
    const std::vector<float*> scales =
        output_scales ? ag_scales(inputs, outputs, to_layers(shard_layers), codec, *output_scales) : std::vector<float*>{};
    const int dt = cgx_dtype(inputs[0]);
    for (int r = 0; r < world_; ++r) {
      for (const at::Tensor* t : {&inputs[r], &outputs[r]})
        TORCH_CHECK(t->is_cuda() && t->is_contiguous() && ((t == &outputs[r] && output_scales) || cgx_dtype(*t) == dt),
                    "bad tensor");
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
                                   (uint64_t)(rs ? outputs[r] : inputs[r]).numel(), ps, rng, streams_[r].stream(), 0,
                                   nullptr, codec, scales.empty() ? nullptr : scales[r]);
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

  // in-place allreduce of one tensor per virtual rank; the prescale is 1/W when averaging unless given
  void allreduce(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, bool average,
                 bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                 std::optional<double> prescale_in, const std::optional<A2aBitsArg>& bits) {
    const auto specs = to_layers(layers);
    const WireCodec codec = allreduce_codec(bits, specs, stochastic);
    if (codec != kMaxMin && kind_ == ReductionType::kAllToAll) throw py::value_error(kAllToAllNoFp8);
    const RngParams rng = make_rng(stochastic, seed, seq);
    const float prescale = sim_prescale(prescale_in, average, hub_.world());
    run(tensors, [&](Reducer& red, int, void* data, int dt, cudaStream_t s) {
      red.allreduce(data, dt, specs, skip_incomplete, prescale, rng, s, codec);
    });
  }
  void broadcast_compressed(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, int root,
                            bool skip_incomplete, bool stochastic, uint64_t seed, uint32_t seq,
                            const std::optional<A2aBitsArg>& bits) {
    TORCH_CHECK(root >= 0 && root < hub_.world(), "LocalReducerGroup: bad root ", root);
    const auto specs = to_layers(layers);
    const WireCodec codec = allreduce_codec(bits, specs, stochastic);
    const RngParams rng = make_rng(stochastic, seed, seq);
    run(tensors, [&](Reducer& red, int, void* data, int dt, cudaStream_t s) {
      red.broadcast_compressed(data, dt, specs, skip_incomplete, root, rng, s, codec);
    });
  }
  // Reducer::reduce_scatter: inputs[r] holds W * S elements, outputs[r] receives shard r
  void reduce_scatter(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs,
                      const std::vector<LayerTuple>& shard_layers, bool average, bool skip_incomplete,
                      bool stochastic, uint64_t seed, uint32_t seq, std::optional<double> prescale_in,
                      const std::optional<A2aBitsArg>& bits) {
    const auto specs = to_layers(shard_layers);
    const WireCodec codec = sharded_codec(bits, specs, stochastic, "reduce_scatter");
    const RngParams rng = make_rng(stochastic, seed, seq);
    const float prescale = sim_prescale(prescale_in, average, hub_.world());
    check_outputs(inputs, outputs, true);
    run(inputs, [&](Reducer& red, int r, void* in, int dt, cudaStream_t s) {
      red.reduce_scatter(in, outputs[r].data_ptr(), dt, specs, skip_incomplete, prescale, rng, s, codec);
    });
  }
  // Reducer::all_gather: inputs[r] holds rank r's shard of S elements, outputs[r] receives W * S
  void all_gather(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs,
                  const std::vector<LayerTuple>& shard_layers, bool skip_incomplete, bool stochastic, uint64_t seed,
                  uint32_t seq, const std::optional<A2aBitsArg>& bits,
                  const std::optional<std::vector<at::Tensor>>& output_scales) {
    const auto specs = to_layers(shard_layers);
    const WireCodec codec = sharded_codec(bits, specs, stochastic, "all_gather");
    const RngParams rng = make_rng(stochastic, seed, seq);
    std::vector<float*> scales;
    if (output_scales)
      scales = ag_scales(inputs, outputs, specs, codec, *output_scales);
    else
      check_outputs(inputs, outputs, false);
    run(inputs, [&](Reducer& red, int r, void* in, int dt, cudaStream_t s) {
      red.all_gather(in, outputs[r].data_ptr(), dt, specs, skip_incomplete, rng, s, codec,
                     scales.empty() ? nullptr : scales[r]);
    });
  }
  // Reducer::all_to_all: counts[q][r] elements go from rank q to r (as LocalSraGroup.all_to_all)
  // Combine, the composed path of the process group (CUDA only): with gate[r], combine_out[r] and
  // output_index[r] (as LocalSraGroup.all_to_all) the received rows land in a scratch buffer, are
  // index_copy_'d into the slots outputs[r] by output_index[r], and combine_rows_kernel writes
  // combine_out[r] from the slots. input_index[r], when given and not None, selects rank r's sent
  // rows of `row` elements from inputs[r] first (index_select, as the process group composes it).
  void all_to_all(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs, const CountMatrix& counts_in,
                  const A2aBitsArg& bits_arg, int64_t bucket, bool stochastic, uint64_t seed, uint32_t seq,
                  const std::optional<std::vector<at::Tensor>>& output_scales, const IndexList& output_index,
                  int64_t row, const IndexList& gate, const IndexList& combine_out, const IndexList& input_index) {
    const A2aBits wb = a2a_bits(bits_arg, stochastic);
    const auto counts = check_counts(counts_in, (size_t)hub_.world());
    TORCH_CHECK_VALUE(input_index.empty() || (row >= 1 && input_index.size() == inputs.size()),
                      "all_to_all: input_index needs row >= 1 and one entry per rank");
    for (size_t r = 0; r < input_index.size(); ++r) {
      const std::optional<at::Tensor>& ix = input_index[r];
      if (!ix) continue;
      TORCH_CHECK_VALUE(ix->device() == inputs[r].device() && ix->scalar_type() == at::kLong && ix->dim() == 1 &&
                            ix->is_contiguous() && inputs[r].is_contiguous() && inputs[r].numel() % row == 0,
                        "all_to_all: rank ", r, "'s input_index must be a contiguous int64 vector on its input's ",
                        "device, and the input whole rows");
      inputs[r] = inputs[r].view({-1, row}).index_select(0, *ix).reshape(-1);
    }
    const std::vector<float*> scales = a2a_scales(output_scales, outputs, wb, bucket);
    check_a2a_tensors(inputs, outputs, counts, inputs[0].is_cuda(), output_scales ? wb.codec : kMaxMin);
    const RngParams rng = make_rng(stochastic, seed, seq);
    const bool combine = !gate.empty() || !combine_out.empty();
    std::vector<A2aRoute> routes((size_t)hub_.world());
    std::vector<at::Tensor> recv;
    if (combine) {
      TORCH_CHECK_VALUE(inputs[0].is_cuda(), "all_to_all: the combine runs on CUDA tensors");
      TORCH_CHECK_VALUE(row >= 1 && output_index.size() == routes.size(), "all_to_all: the combine needs row >= 1 ",
                        "and one output_index per rank");
      for (size_t r = 0; r < routes.size(); ++r) {
        const std::optional<at::Tensor>& ix = output_index[r];
        TORCH_CHECK_VALUE(ix && ix->is_cuda() && ix->scalar_type() == at::kLong && ix->dim() == 1 &&
                              ix->is_contiguous() && ix->numel() * row == outputs[r].numel(),
                          "all_to_all: rank ", r, "'s output_index must be a contiguous CUDA int64 vector of one ",
                          "entry per row of its output");
        routes[r].out_index = ix->data_ptr<int64_t>();
        routes[r].row = (uint64_t)row;
        routes[r].out_rows = (uint64_t)ix->numel();
        recv.push_back(at::empty_like(outputs[r]));
      }
      combine_routes(routes, inputs, gate, combine_out, wb, bucket, row, output_scales.has_value());
    }
    run(inputs, [&](Reducer& red, int r, void* in, int dt, cudaStream_t s) {
      std::vector<uint64_t> out_counts(counts.size());
      for (size_t q = 0; q < counts.size(); ++q) out_counts[q] = counts[q][r];
      red.all_to_all(in, combine ? recv[r].data_ptr() : outputs[r].data_ptr(), counts[r], out_counts, dt, wb.bits,
                     wb.codec, (uint32_t)bucket, rng, s, scales.empty() ? nullptr : scales[r]);
    }, false);
    for (size_t r = 0; combine && r < routes.size(); ++r) {
      outputs[r].view({-1, row}).index_copy_(0, *output_index[r], recv[r].view({-1, row}));
      if (routes[r].topk == 0) continue;
      cuda_check(launch_combine_rows(outputs[r].data_ptr(), routes[r].gate, routes[r].combine_out,
                                     cgx_dtype(inputs[r]), routes[r].out_rows / routes[r].topk, routes[r].topk,
                                     (uint32_t)row, c10::cuda::getCurrentCUDAStream().stream()),
                 "launch_combine_rows");
    }
  }
  // bytes each rank's reducer counted as sent during the last call
  std::vector<int64_t> bytes_sent() const { return last_sent_; }
  // plans cached by rank r's reducer, and tables it has uploaded so far, on the backend (host or
  // device memory) of the last call
  int64_t num_plans(int r) { return (int64_t)rank_of_last_call(r).red->num_plans(); }
  int64_t plan_uploads(int r) { return (int64_t)rank_of_last_call(r).red->plan_uploads(); }
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

  Rank& rank_of_last_call(int r) {
    TORCH_CHECK(r >= 0 && r < hub_.world(), "LocalReducerGroup: bad rank ", r);
    return ranks(last_cuda_)[(size_t)r];
  }

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

  // one output per rank, contiguous, of the inputs' dtype and device, holding S (reduce-scatter) or
  // W * S elements (all-gather) for inputs of W * S or S
  void check_outputs(const std::vector<at::Tensor>& inputs, const std::vector<at::Tensor>& outputs, bool rs) const {
    const int64_t W = hub_.world();
    TORCH_CHECK(inputs.size() == outputs.size(), "LocalReducerGroup: one output per input");
    for (size_t r = 0; r < inputs.size(); ++r) {
      const at::Tensor &i = inputs[r], &o = outputs[r];
      TORCH_CHECK(o.is_contiguous() && o.scalar_type() == i.scalar_type() && o.device() == i.device() &&
                      (rs ? i.numel() == o.numel() * W : o.numel() == i.numel() * W),
                  "LocalReducerGroup: contiguous outputs of the inputs' dtype and device, ",
                  rs ? "inputs of W * S and outputs of S elements" : "inputs of S and outputs of W * S elements");
    }
  }

  // same_size false: the ranks' tensors may differ in size (all_to_all)
  template <class F>
  void run(const std::vector<at::Tensor>& tensors, F&& op, bool same_size = true) {
    const int W = hub_.world();
    TORCH_CHECK((int)tensors.size() == W, "LocalReducerGroup: need one tensor per virtual rank (", W, "), got ",
                tensors.size());
    const int dt = cgx_dtype(tensors[0]);
    const bool cuda = tensors[0].is_cuda();
    for (const at::Tensor& t : tensors)
      TORCH_CHECK(t.is_contiguous() && cgx_dtype(t) == dt && (!same_size || t.numel() == tensors[0].numel()) &&
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
    last_cuda_ = cuda;
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
            op(*rk[r].red, r, tensors[r].data_ptr(), dt, s);
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
  bool last_cuda_ = false;
  int device_ = -1;
  std::vector<c10::cuda::CUDAStream> streams_;
  std::vector<Rank> cpu_, cuda_;
  std::vector<int64_t> last_sent_;
};

// W AllreduceEngines in one process, `local_size` consecutive virtual ranks per node, wired as
// ProcessGroupCGX wires them: per node a set of connect_local heaps (the fused kernels) and one
// loopback hub (the generic intra-node reducers and broadcasts), per local rank one loopback hub
// across the nodes (the cross-node reducers), for host and for device memory. Each rank's call runs
// on its own host thread and stream. An observer logs every stage the engine issues, and before a
// fused launch waits until every rank of the node has reached the same launch: the ranks share one
// CUDA context, where one rank's plan upload or cudaFree can wait for a peer's kernel that spins
// until this rank launches.
class LocalEngineGroup {
 public:
  LocalEngineGroup(int world, int local_size, const py::dict& config, int lanes, int64_t slot_bytes,
                   int64_t timeout_ms)
      : world_(world), local_size_(local_size), nodes_(local_size >= 1 ? world / local_size : 1) {
    TORCH_CHECK(world >= 1 && world <= kA2aMaxWorld, "LocalEngineGroup: world must be 1..", kA2aMaxWorld, ", got ", world);
    TORCH_CHECK(local_size >= 1 && world % local_size == 0, "LocalEngineGroup: local_size ", local_size,
                " does not divide the world ", world);
    // streams r and r + 8 share a hardware queue: a rank's kernel could wait behind a peer's that spins for it
    TORCH_CHECK(local_size <= 8, "LocalEngineGroup: at most 8 ranks per node, got ", local_size);
    TORCH_CHECK(lanes >= 1, "LocalEngineGroup: lanes must be positive");
    EngineConfig cfg = EngineConfig::read();
    cfg.timeout_ms = timeout_ms;
    cfg.lanes = lanes;
    cfg.local_size = local_size;
    bool p2p = true;
    for (const auto& kv : config) {
      const std::string k = py::cast<std::string>(kv.first);
      const py::handle v = kv.second;
      if (k == "fusion_bytes") cfg.fusion_bytes = py::cast<int64_t>(v);
      else if (k == "oneshot_max_bytes") cfg.oneshot_max_bytes = py::cast<int64_t>(v);
      else if (k == "min_lane_elems") cfg.min_lane_elems = py::cast<uint32_t>(v);
      else if (k == "min_compress_elems") cfg.min_compress_elems = py::cast<int>(v);
      else if (k == "inner_reduction") cfg.inner_reduction = reduction(py::cast<std::string>(v));
      else if (k == "cross_reduction") cfg.cross_reduction = reduction(py::cast<std::string>(v));
      else if (k == "intra_broadcast") cfg.intra_broadcast = py::cast<bool>(v);
      else if (k == "intra_compress") cfg.intra_compress = py::cast<bool>(v);
      else if (k == "dummy_compression") cfg.dummy_compression = py::cast<bool>(v);
      else if (k == "overlap_lanes") cfg.overlap_lanes = py::cast<int>(v);
      else if (k == "p2p") p2p = py::cast<bool>(v);
      else TORCH_CHECK(false, "LocalEngineGroup: unknown config key '", k, "'");
    }
    // without heaps the intra-node stage runs the generic reducers
    cfg.inner_comm = p2p ? CommType::kP2P : CommType::kNCCL;
    cfg.fake_ratio = 1.0;
    const int nodes = world / local_size;
    if (p2p) {
      // every heap's CTAs spin on their peers': all of them must be resident at once, with room to
      // spare for the generic reducers' kernels. The nodes' kernels run side by side on this one GPU.
      int resident = std::numeric_limits<int>::max();
      for (int dt : {kF32, kF16, kBF16}) resident = std::min(resident, sra_max_resident_ctas(dt));
      TORCH_CHECK((int64_t)world * lanes <= resident / 2, "LocalEngineGroup: ", world, " ranks x ", lanes,
                  " lanes cannot all be resident (", resident, " CTAs, half of them usable)");
      TORCH_CHECK(cudaGetDevice(&device_) == cudaSuccess, "LocalEngineGroup: no CUDA device");
    }
    for (int n = 0; n < nodes; ++n) intra_hubs_.push_back(std::make_unique<LoopbackHub>(local_size, timeout_ms));
    for (int l = 0; l < local_size; ++l) cross_hubs_.push_back(std::make_unique<LoopbackHub>(nodes, timeout_ms));
    world_hub_ = std::make_unique<LoopbackHub>(world, timeout_ms);
    a2a_hub_ = std::make_unique<LoopbackHub>(world, timeout_ms);
    for (int r = 0; r < world; ++r) {
      auto e = std::make_unique<AllreduceEngine>(r, world, cfg);
      e->set_topology(local_size);
      for (bool cuda : {false, true}) {
        std::unique_ptr<Communicator> intra, cross;
        if (local_size > 1) intra = std::make_unique<LoopbackCommunicator>(intra_hub(r), e->local_rank(), cuda);
        if (nodes > 1) cross = std::make_unique<LoopbackCommunicator>(cross_hub(r), e->node(), cuda);
        e->attach_generic(cuda, std::move(intra), std::move(cross));
      }
      // the all-to-all's cross-node exchange, as the process group's CUDA delegate carries it
      if (nodes > 1) e->attach_world(true, std::make_unique<LoopbackCommunicator>(a2a_hub_.get(), r, true));
      engines_.push_back(std::move(e));
      observers_.push_back(std::make_unique<Observer>(this, r));
      engines_[r]->set_observer(observers_[r].get());
    }
    if (p2p) {
      layout_ = HeapLayout::make(local_size, lanes, (size_t)slot_bytes,
                                 AllreduceEngine::required_oneshot_slot_bytes(cfg));
      for (int n = 0; n < nodes; ++n) {
        std::vector<std::unique_ptr<SymmetricHeap>> heaps;
        std::vector<SymmetricHeap*> all;
        for (int l = 0; l < local_size; ++l) {
          heaps.push_back(std::make_unique<SymmetricHeap>(l, local_size, layout_));
          all.push_back(heaps.back().get());
        }
        for (auto& h : heaps) h->connect_local(all);
        for (int l = 0; l < local_size; ++l) engines_[n * local_size + l]->attach_heap(std::move(heaps[l]), lanes);
      }
    }
  }
  ~LocalEngineGroup() {
    std::optional<c10::cuda::CUDAGuard> g;
    if (device_ >= 0) g.emplace((c10::DeviceIndex)device_);
    engines_.clear();
  }

  // `bits`, when given, is the wire format of the 8-bit layers (a2a_bits: an FP8 name, or an integer
  // for max-min) in place of CGX_COMPRESSION_FORMAT's; the widths stay the environment's / the table's
  void allreduce(std::vector<at::Tensor> tensors, bool average, int explicit_bucket, bool overlapped,
                 const std::optional<A2aBitsArg>& bits) {
    const std::optional<WireCodec> codec = format_of(bits);
    run(tensors, [&](AllreduceEngine& e, int, void* data, int dt, int64_t n, bool cuda, cudaStream_t s) {
      if (cuda) {
        e.allreduce_cuda(data, dt, n, average, explicit_bucket, s, overlapped, codec);
      } else {
        AllreduceEngine::CpuCall call = e.prepare_cpu(n, explicit_bucket);
        if (codec) call.env.codec = *codec;
        e.allreduce_cpu_prepared(data, dt, call, average);
      }
    });
  }
  void allreduce_layers(std::vector<at::Tensor> tensors, const std::vector<LayerTuple>& layers, bool average,
                        const std::optional<A2aBitsArg>& bits) {
    const auto specs = to_layers(layers);
    const std::optional<WireCodec> codec = format_of(bits);
    run(tensors, [&](AllreduceEngine& e, int, void* data, int dt, int64_t, bool cuda, cudaStream_t s) {
      AllreduceEngine::CpuCall call;
      call.env = CompressionEnv::read();
      if (codec) call.env.codec = *codec;
      call.layers = specs;
      if (cuda)
        e.allreduce_cuda_layers(data, dt, specs, average, call.env, s);
      else
        e.allreduce_cpu_prepared(data, dt, call, average);
    });
  }
  // inputs[r] / outputs[r]: rank r's buffers of the reduce-scatter (W * S -> S) or the all-gather
  // (S -> W * S); `shard_layers` is one shard's table, by default one layer of S elements with the
  // environment's width and bucket size. Host tensors run the generic reducers (no heaps). The
  // all-gather runs without skip_incomplete, as the process group's does. `bits`, when given,
  // replaces the environment's width: an integer, or an FP8 format name (a2a_bits; the table's
  // layers then need bits 8 or 32).
  // With output_scales (all-gather, an FP8 `bits`): the codes output (ag_scales), the table by
  // default one 8-bit layer with the environment's bucket size.
  void sharded(bool reduce_scatter, std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs, bool average,
               const std::optional<std::vector<LayerTuple>>& shard_layers, const std::optional<A2aBitsArg>& bits,
               const std::optional<std::vector<at::Tensor>>& output_scales = std::nullopt) {
    const ShardedOp op = reduce_scatter ? ShardedOp::kReduceScatter : ShardedOp::kAllGather;
    TORCH_CHECK((int)outputs.size() == world_, "LocalEngineGroup: one output per virtual rank");
    CompressionEnv env = CompressionEnv::read();
    WireCodec codec = kMaxMin;
    if (bits) {
      const A2aBits wb = a2a_bits(*bits, env.stochastic, op_name(op));
      env.bits = wb.bits;
      codec = sharded_codec(bits, shard_layers ? to_layers(*shard_layers) : std::vector<LayerSpec>{},
                            env.stochastic, op_name(op));
    }
    const bool skip = reduce_scatter && env.skip_incomplete;
    RngParams rng = make_rng(env.stochastic, env.seed, 0);
    const std::vector<LayerSpec> given = shard_layers ? to_layers(*shard_layers) : std::vector<LayerSpec>{};
    std::vector<float*> scales;
    if (output_scales) {
      const int64_t S = inputs.empty() ? 0 : inputs[0].numel();
      scales = ag_scales(inputs, outputs,
                         shard_layers ? given : std::vector<LayerSpec>{LayerSpec{0, (uint64_t)S, 8, (uint32_t)env.bucket_size}},
                         codec, *output_scales);
    }
    run(inputs, [&](AllreduceEngine& e, int r, void* in, int dt, int64_t n, bool cuda, cudaStream_t s) {
      TORCH_CHECK(outputs[r].is_contiguous() && (!scales.empty() || cgx_dtype(outputs[r]) == dt) &&
                      outputs[r].device() == inputs[r].device(),
                  "LocalEngineGroup: contiguous outputs of the inputs' dtype and device");
      TORCH_CHECK(cuda || !e.fused(), "LocalEngineGroup: host tensors need a group without heaps (p2p=False)");
      const int64_t S = reduce_scatter ? outputs[r].numel() : n;
      TORCH_CHECK((reduce_scatter ? n : outputs[r].numel()) == S * world_, "LocalEngineGroup: the full buffer holds W x S");
      const std::vector<LayerSpec> table =
          scales.empty() || shard_layers ? e.sharded_table(S, given, env.bits, env.bucket_size)
                                         : std::vector<LayerSpec>{LayerSpec{0, (uint64_t)S, 8, (uint32_t)env.bucket_size}};
      at::Tensor staging;
      if (const int64_t sn = e.sharded_staging_numel(S)) staging = at::empty({sn}, inputs[r].options());
      // upload every window's plan and wait for it before any rank launches (see the class comment)
      if (e.fused()) {
        e.prepare_sharded(op, table, dt, skip, s);
        cuda_check(cudaStreamSynchronize(s), "LocalEngineGroup: plan upload");
        intra_hub(r)->barrier(e.local_rank());
      }
      e.sharded(cuda, op, in, outputs[r].data_ptr(), staging.defined() ? staging.data_ptr() : nullptr, dt, S, table,
                average, skip, rng, s, false, codec, scales.empty() ? nullptr : scales[r]);
      // the staging buffer is freed on the caller's stream when this returns: let its work finish first
      if (staging.defined() && cuda) cuda_check(cudaStreamSynchronize(s), "LocalEngineGroup: sharded call");
    });
  }

  // inputs[r] / outputs[r]: rank r's compressed all-to-all (AllreduceEngine::all_to_all), counts[q][r]
  // elements from rank q to rank r; with output_scales (an FP8 `bits`) the codes output. A call's
  // stochastic streams use the sequence number the engine gives it, which log(r) reports on several
  // nodes. Routed forms (any of input_index, output_index, input_scale, gate with combine_out given
  // for some rank; tensors of rows of `row` elements, the counts those of the logical buffers) run
  // as the process group runs them when the fused kernel does not route the rows: a2a_compose.
  void all_to_all(std::vector<at::Tensor> inputs, std::vector<at::Tensor> outputs, const CountMatrix& counts_in,
                  const A2aBitsArg& bits_arg, int64_t bucket, bool stochastic, uint64_t seed,
                  const std::optional<std::vector<at::Tensor>>& output_scales, const IndexList& input_index,
                  const IndexList& output_index, const IndexList& input_scale, const IndexList& gate,
                  const IndexList& combine_out, int64_t row) {
    const A2aBits wb = a2a_bits(bits_arg, stochastic);
    const auto counts = check_counts(counts_in, (size_t)world_);
    TORCH_CHECK((int)inputs.size() == world_ && (int)outputs.size() == world_,
                "LocalEngineGroup: one input and one output per virtual rank");
    const std::vector<float*> scales = a2a_scales(output_scales, outputs, wb, bucket);
    const RngParams rng = make_rng(stochastic, seed, 0);
    auto opt = [&](const IndexList& l, int r) {
      TORCH_CHECK(l.empty() || (int)l.size() == world_, "LocalEngineGroup: one entry per virtual rank or none");
      return l.empty() || !l[r] ? at::Tensor() : *l[r];
    };
    bool routed = false;
    for (const IndexList* l : {&input_index, &output_index, &input_scale, &gate, &combine_out})
      for (const auto& t : *l) routed |= t.has_value();
    if (!routed) {
      check_a2a_tensors(inputs, outputs, counts, inputs[0].is_cuda(), output_scales ? wb.codec : kMaxMin);
      run(inputs,
          [&](AllreduceEngine& e, int r, void* in, int dt, int64_t, bool cuda, cudaStream_t s) {
            std::vector<uint64_t> out_counts(world_);
            for (int q = 0; q < world_; ++q) out_counts[q] = counts[q][r];
            e.all_to_all(cuda, in, outputs[r].data_ptr(), counts[r], out_counts, dt, wb.bits, wb.codec,
                         (uint32_t)bucket, rng, s, nullptr, scales.empty() ? nullptr : scales[r]);
          },
          false);
      return;
    }
    TORCH_CHECK(row >= 1, "LocalEngineGroup: row must be >= 1");
    for (int r = 0; r < world_; ++r) {
      uint64_t nin = 0, nout = 0;
      for (int q = 0; q < world_; ++q) {
        nin += counts[r][q];
        nout += counts[q][r];
      }
      const at::Tensor ii = opt(input_index, r), oi = opt(output_index, r);
      TORCH_CHECK(inputs[r].is_cuda() && outputs[r].is_cuda() && inputs[r].dim() == 2 && outputs[r].dim() == 2 &&
                      inputs[r].size(1) == row && outputs[r].size(1) == row,
                  "LocalEngineGroup: routed calls take CUDA tensors [rows, row]");
      TORCH_CHECK((uint64_t)(ii.defined() ? ii.numel() : inputs[r].size(0)) * (uint64_t)row == nin &&
                      (uint64_t)(oi.defined() ? oi.numel() : outputs[r].size(0)) * (uint64_t)row == nout,
                  "all_to_all: rank ", r, "'s tensors do not match its row and column of the counts");
    }
    run(inputs,
        [&](AllreduceEngine& e, int r, void*, int dt, int64_t, bool, cudaStream_t s) {
          std::vector<uint64_t> out_counts(world_);
          for (int q = 0; q < world_; ++q) out_counts[q] = counts[q][r];
          c10::cuda::CUDAStreamGuard sg(streams_[r]);
          const at::Tensor sc = scales.empty() ? at::Tensor() : (*output_scales)[r].view({outputs[r].size(0), -1});
          a2a_compose(e, inputs[r], outputs[r], counts[r], out_counts, dt, wb.bits, wb.codec, (uint32_t)bucket, rng,
                      opt(input_index, r), opt(output_index, r), opt(input_scale, r), sc, opt(gate, r),
                      opt(combine_out, r), s);
        },
        false);
  }

  py::dict stats(int r) const {
    TORCH_CHECK(r >= 0 && r < world_, "LocalEngineGroup: bad rank ", r);
    const EngineStats& s = engines_[r]->stats();
    py::dict d;
    d["calls"] = s.calls;
    d["kernel_launches"] = s.kernel_launches;
    d["elements"] = s.elements;
    d["wire_bytes"] = s.wire_bytes;
    d["raw_bytes"] = s.raw_bytes;
    return d;
  }
  void check() {
    for (auto& e : engines_) e->check_health();
  }
  // the stages rank r issued in the last call, in order
  py::list log(int r) const {
    TORCH_CHECK(r >= 0 && r < world_, "LocalEngineGroup: bad rank ", r);
    py::list out;
    for (const Entry& e : observers_[r]->log) {
      py::dict d;
      d["kind"] = e.kind;
      d["layers"] = e.layers;
      d["lanes"] = e.lanes;
      d["numel"] = e.numel;
      d["seed"] = e.seed;
      d["seq"] = e.seq;
      d["stochastic"] = e.stochastic;
      d["scale"] = e.scale;
      out.append(d);
    }
    return out;
  }
  // (slot bytes, one-shot slot bytes) of the heaps; (0, 0) without them
  std::pair<int64_t, int64_t> slot_bytes() const {
    return {(int64_t)layout_.slot_bytes, (int64_t)layout_.os_slot_bytes};
  }
  int64_t num_plans(int r) const {
    TORCH_CHECK(r >= 0 && r < world_, "LocalEngineGroup: bad rank ", r);
    return engines_[r]->fused() ? (int64_t)engines_[r]->fused()->num_plans() : 0;
  }

 private:
  struct Entry {
    std::string kind;
    std::vector<LayerTuple> layers;
    int64_t lanes = 0, numel = 0;
    uint64_t seed = 0;
    uint32_t seq = 0;
    bool stochastic = false;
    float scale = 1.0f;
  };
  struct Observer : EngineObserver {
    Observer(LocalEngineGroup* g, int r) : group(g), rank(r) {}
    void before_fused_launch(const DevicePlan&, cudaStream_t stream) override {
      FusedSra* f = group->engines_[rank]->fused();
      if (f->num_plans() != plans_seen || f->generation() != generation_seen) {
        cuda_check(cudaStreamSynchronize(stream), "LocalEngineGroup: plan upload");
        plans_seen = f->num_plans();
        generation_seen = f->generation();
      }
      group->intra_hub(rank)->barrier(group->engines_[rank]->local_rank());
    }
    void stage(const EngineStage& s) override {
      static const char* kNames[] = {"oneshot", "sra",     "generic_intra", "cross",      "bcast_compressed", "bcast_raw",
                                     "rs",      "ag",      "generic_rs",    "generic_ag", "cross_rs",         "cross_ag",
                                     "a2a_cross", "a2a_intra"};
      // A sharded call over several nodes runs fused launches next to generic stages, whose
      // cudaMalloc / cudaFree can wait for a fused kernel of another node that spins for a peer the
      // same driver call holds up. Every rank issues the same sharded stages, so before each of them
      // all ranks drain their streams and meet: no fused kernel runs while a generic stage does.
      if (s.a2a() && group->nodes_ > 1) {
        // The all-to-all's node-local stages run one node at a time, in node order: with more than
        // eight ranks two nodes' spinning kernels can share hardware queues, each behind the other.
        // Node n meets n + 1 times before its stage (round 0 drains the pack) and N - n times after it,
        // once its stream has drained; round t lets node t start after node t - 1 has finished.
        const int n = rank / group->local_size_, N = group->nodes_;
        const int rounds = s.kind == EngineStage::kA2aIntra ? n + 1 : N - n;
        for (int t = 0; t < rounds; ++t) {
          if (group->call_cuda_ && (t == 0 || s.kind == EngineStage::kA2aIntra))
            cuda_check(cudaStreamSynchronize(group->streams_[rank].stream()), "LocalEngineGroup: quiesce");
          group->world_hub_->barrier(rank);
        }
      } else if (s.sharded() && group->nodes_ > 1) {
        if (group->call_cuda_)
          cuda_check(cudaStreamSynchronize(group->streams_[rank].stream()), "LocalEngineGroup: quiesce");
        group->world_hub_->barrier(rank);
      }
      Entry e;
      e.kind = kNames[s.kind];
      if (s.layers)
        for (const LayerSpec& l : *s.layers)
          e.layers.emplace_back((int64_t)l.elem_off, (int64_t)l.numel, (int64_t)l.bits, (int64_t)l.bucket);
      if (s.dp) {
        e.lanes = s.dp->plan.lanes;
        e.numel = (int64_t)s.dp->plan.numel;
      } else {
        for (const LayerSpec& l : *s.layers) e.numel += (int64_t)l.numel;
      }
      e.seed = s.rng.seed;
      e.seq = s.rng.seq;
      e.stochastic = s.rng.stochastic;
      e.scale = s.scale;
      log.push_back(std::move(e));
    }
    LocalEngineGroup* group;
    int rank;
    size_t plans_seen = 0;
    uint64_t generation_seen = 0;
    std::vector<Entry> log;
  };

  static std::optional<WireCodec> format_of(const std::optional<A2aBitsArg>& bits) {
    if (!bits) return std::nullopt;
    return a2a_bits(*bits, CompressionEnv::read().stochastic, "allreduce").codec;
  }
  static ReductionType reduction(const std::string& k) {
    if (k == "SRA") return ReductionType::kSRA;
    if (k == "RING") return ReductionType::kRing;
    if (k == "ALLTOALL") return ReductionType::kAllToAll;
    TORCH_CHECK(false, "LocalEngineGroup: a reduction is SRA, RING or ALLTOALL, got ", k);
    return ReductionType::kSRA;
  }
  LoopbackHub* intra_hub(int r) const { return intra_hubs_[r / local_size_].get(); }
  LoopbackHub* cross_hub(int r) const { return cross_hubs_[r % local_size_].get(); }
  void fail_all(const std::string& msg) {
    for (auto& h : intra_hubs_) h->fail(msg);
    for (auto& h : cross_hubs_) h->fail(msg);
    world_hub_->fail(msg);
    a2a_hub_->fail(msg);
  }

  // op(engine, rank, data, dtype, numel, cuda, stream) on every rank's thread; every rank's stream is
  // synchronised before this returns, and the first failure of any rank is raised
  // (same_size false: the tensors may differ in size)
  template <class F>
  void run(const std::vector<at::Tensor>& tensors, F&& op, bool same_size = true) {
    const int W = world_;
    TORCH_CHECK((int)tensors.size() == W, "LocalEngineGroup: need one tensor per virtual rank (", W, "), got ",
                tensors.size());
    const int dt = cgx_dtype(tensors[0]);
    const bool cuda = tensors[0].is_cuda();
    for (const at::Tensor& t : tensors)
      TORCH_CHECK(t.is_contiguous() && cgx_dtype(t) == dt && (!same_size || t.numel() == tensors[0].numel()) &&
                      t.device() == tensors[0].device(),
                  "LocalEngineGroup: contiguous tensors of one dtype, size and device");
    TORCH_CHECK(cuda || tensors[0].device().is_cpu(), "LocalEngineGroup: CPU or CUDA tensors");
    c10::cuda::OptionalCUDAGuard guard;
    if (cuda) {
      const int dev = tensors[0].device().index();
      TORCH_CHECK(device_ < 0 || device_ == dev, "LocalEngineGroup: all calls use one device (", device_, ")");
      device_ = dev;
      guard.set_index((c10::DeviceIndex)device_);
      if (streams_.empty())
        for (int r = 0; r < W; ++r) streams_.push_back(c10::cuda::getStreamFromPool(false, (c10::DeviceIndex)device_));
      at::cuda::CUDAEvent ready(cudaEventDisableTiming);
      ready.record(c10::cuda::getCurrentCUDAStream());
      for (auto& s : streams_) ready.block(s);
    }
    for (auto& h : intra_hubs_) h->reset(false);
    for (auto& h : cross_hubs_) h->reset(false);
    world_hub_->reset(false);
    a2a_hub_->reset(false);
    call_cuda_ = cuda;
    for (auto& o : observers_) o->log.clear();
    const int64_t n = tensors[0].numel();
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
            op(*engines_[r], r, tensors[r].data_ptr(), dt, n, cuda, s);
            if (cuda) cuda_check(cudaStreamSynchronize(s), "LocalEngineGroup: synchronise a virtual rank");
          } catch (const std::exception& e) {
            fail_all("rank " + std::to_string(r) + ": " + e.what());
          } catch (...) {
            fail_all("rank " + std::to_string(r) + ": unknown exception");
          }
          intra_hub(r)->finish(engines_[r]->local_rank());
          cross_hub(r)->finish(engines_[r]->node());
          world_hub_->finish(r);
          a2a_hub_->finish(r);
        });
      for (auto& t : threads) t.join();
      // a rank that threw skipped its own synchronise: nothing it queued may run on after this returns
      if (cuda)
        for (int r = 0; r < W; ++r) {
          const cudaError_t err = cudaStreamSynchronize(streams_[r].stream());
          if (err != cudaSuccess)
            fail_all("rank " + std::to_string(r) + ": synchronise after the call: " + cudaGetErrorString(err));
        }
    }
    for (auto& h : intra_hubs_) TORCH_CHECK(!h->failed(), "LocalEngineGroup: ", h->failure());
    for (auto& h : cross_hubs_) TORCH_CHECK(!h->failed(), "LocalEngineGroup: ", h->failure());
    TORCH_CHECK(!world_hub_->failed(), "LocalEngineGroup: ", world_hub_->failure());
    TORCH_CHECK(!a2a_hub_->failed(), "LocalEngineGroup: ", a2a_hub_->failure());
    if (cuda) check();
  }

  int world_, local_size_, nodes_;
  int device_ = -1;
  bool call_cuda_ = false;  // the running call's tensors are device memory
  HeapLayout layout_{};
  std::vector<std::unique_ptr<LoopbackHub>> intra_hubs_, cross_hubs_;
  std::unique_ptr<LoopbackHub> world_hub_;  // barriers of every rank (Observer::stage)
  std::unique_ptr<LoopbackHub> a2a_hub_;    // the all-to-all's cross-node exchange
  std::vector<std::unique_ptr<AllreduceEngine>> engines_;  // after the hubs: released first
  std::vector<std::unique_ptr<Observer>> observers_;
  std::vector<c10::cuda::CUDAStream> streams_;
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
// candidate width (engine/quant_error_table.h)
at::Tensor py_quantization_error(const at::Tensor& t, const std::vector<LayerTuple>& layers,
                                 const std::vector<int64_t>& candidates, bool stochastic, double prescale,
                                 bool skip_incomplete, int64_t chunks, int64_t skip_chunk) {
  std::vector<QErrSpan> spans;
  spans.reserve(layers.size());
  for (const auto& l : layers) spans.push_back({std::get<0>(l), std::get<1>(l), std::get<3>(l)});
  return quantization_error_table(t, spans, candidates, stochastic, prescale, skip_incomplete, chunks, skip_chunk);
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
      .def(
          "allreduce_bucket",
          [](ProcessGroupCGX& pg, at::Tensor& tensor, int64_t bucket_idx, bool average,
             const std::optional<A2aBitsArg>& bits) {
            // an FP8 name replaces CGX_COMPRESSION_FORMAT's wire format; the widths stay the registry's
            std::optional<WireCodec> codec;
            if (bits) codec = a2a_bits(*bits, CompressionEnv::read().stochastic, "allreduce").codec;
            py::gil_scoped_release nogil;
            return pg.allreduce_bucket(tensor, bucket_idx, average, codec);
          },
          py::arg("tensor"), py::arg("bucket_idx"), py::arg("average") = false, py::arg("bits") = py::none())
      .def("reduce_scatter_compressed",
           [](ProcessGroupCGX& pg, at::Tensor out, at::Tensor in, bool average, const A2aBitsArg& bits,
              int bucket_size, bool skip_incomplete, bool stochastic, int64_t seed, bool overlapped,
              const std::vector<LayerTuple>& layers) {
             const auto table = to_layers(layers);
             const A2aBits wb = a2a_bits(bits, stochastic, "reduce_scatter");
             sharded_codec(bits, table, stochastic, "reduce_scatter");
             return pg.sharded_compressed(ShardedOp::kReduceScatter, out, in, average, wb.bits, wb.codec, bucket_size,
                                          skip_incomplete, stochastic, seed, overlapped, table);
           },
           py::arg("output"), py::arg("input"), py::arg("average") = false, py::arg("bits") = 4,
           py::arg("bucket_size") = 512, py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
           py::arg("seed") = -1, py::arg("overlapped") = false, py::arg("layers") = std::vector<LayerTuple>{},
           py::call_guard<py::gil_scoped_release>())
      .def("all_gather_compressed",
           [](ProcessGroupCGX& pg, at::Tensor out, at::Tensor in, const A2aBitsArg& bits, int bucket_size,
              bool stochastic, int64_t seed, bool overlapped, const std::vector<LayerTuple>& layers,
              const std::optional<at::Tensor>& out_scales) {
             const auto table = to_layers(layers);
             const A2aBits wb = a2a_bits(bits, stochastic, "all_gather");
             sharded_codec(bits, table, stochastic, "all_gather");
             return pg.sharded_compressed(ShardedOp::kAllGather, out, in, false, wb.bits, wb.codec, bucket_size, false,
                                          stochastic, seed, overlapped, table, out_scales.value_or(at::Tensor()));
           },
           py::arg("output"), py::arg("input"), py::arg("bits") = 4, py::arg("bucket_size") = 512,
           py::arg("stochastic") = false, py::arg("seed") = -1, py::arg("overlapped") = false,
           py::arg("layers") = std::vector<LayerTuple>{}, py::arg("output_scales") = py::none(),
           py::call_guard<py::gil_scoped_release>())
      .def("all_to_all_compressed",
           [](ProcessGroupCGX& pg, at::Tensor out, at::Tensor in, const std::vector<int64_t>& out_splits,
              const std::vector<int64_t>& in_splits, const A2aBitsArg& bits, int bucket_size, bool stochastic,
              int64_t seed, const std::optional<at::Tensor>& in_index, const std::optional<at::Tensor>& out_index,
              const std::optional<at::Tensor>& out_scales, const std::optional<at::Tensor>& gate,
              const std::optional<at::Tensor>& combine_out, const std::optional<at::Tensor>& in_scale) {
             const A2aBits wb = a2a_bits(bits, stochastic);
             return pg.all_to_all_compressed(out, in, out_splits, in_splits, wb.bits, wb.codec, bucket_size,
                                             stochastic, seed, in_index.value_or(at::Tensor()),
                                             out_index.value_or(at::Tensor()), out_scales.value_or(at::Tensor()),
                                             gate.value_or(at::Tensor()), combine_out.value_or(at::Tensor()),
                                             in_scale.value_or(at::Tensor()));
           },
           py::arg("output"), py::arg("input"), py::arg("output_split_sizes") = std::vector<int64_t>{},
           py::arg("input_split_sizes") = std::vector<int64_t>{}, py::arg("bits") = 8, py::arg("bucket_size") = 512,
           py::arg("stochastic") = false, py::arg("seed") = -1, py::arg("input_index") = py::none(),
           py::arg("output_index") = py::none(), py::arg("output_scales") = py::none(),
           py::arg("gate") = py::none(), py::arg("combine_out") = py::none(), py::arg("input_scale") = py::none(),
           py::call_guard<py::gil_scoped_release>())
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

  using Assignment = std::map<std::pair<int64_t, int64_t>, int>;
  py::class_<HookState, std::shared_ptr<HookState>>(m, "NativeHookState")
      .def_property_readonly("step", [](const HookState& h) { return h.step.load(); })
      .def_readonly("layer_min_size", &HookState::layer_min_size)
      .def_readonly("bits", &HookState::bits)
      .def_readonly("bucket_size", &HookState::bucket_size)
      .def_readonly("register_step", &HookState::register_step)
      .def_readonly("candidates", &HookState::candidates)
      .def_readonly("period", &HookState::period)
      // (bucket, layer) -> width applied by a decision or a loaded assignment
      .def_property_readonly("assignment", [](HookState& h) {
        std::lock_guard<std::mutex> lk(h.mu);
        return h.assignment;
      })
      // group-summed [rows, candidates] float64 table of the last decision, or None
      .def_property_readonly("last_errors", [](HookState& h) -> std::optional<at::Tensor> {
        std::lock_guard<std::mutex> lk(h.mu);
        if (!h.last_errors.defined()) return std::nullopt;
        return h.last_errors;
      })
      // (bucket, layer, elem_off, numel) of every adapted layer, in bucket order
      .def_property_readonly("adapted_layers", [](HookState& h) {
        std::vector<std::tuple<int64_t, int64_t, int64_t, int64_t>> out;
        for (const AdaptedLayer& l : h.adapted_layers()) out.emplace_back(l.bucket, l.layer, l.elem_off, l.numel);
        return out;
      })
      // widths to apply when the layers are registered (a checkpoint's assignment)
      .def("load_assignment", [](HookState& h, const Assignment& a) {
        std::lock_guard<std::mutex> lk(h.mu);
        h.loaded = a;
      }, py::arg("assignment"));
  m.def("register_native_hook",
        [](const std::shared_ptr<c10d::Reducer>& reducer, const c10::intrusive_ptr<ProcessGroupCGX>& pg,
           int64_t layer_min_size, const A2aBitsArg& bits, int bucket_size, int register_step,
           std::vector<int64_t> candidates, int64_t period, Assignment assignment) {
          // an FP8 name: layers registered at 8 bits, sent in that format
          const A2aBits wb = a2a_bits(bits, false, "allreduce");
          std::optional<WireCodec> codec;
          if (wb.codec != kMaxMin) codec = wb.codec;
          return register_native_hook(reducer, pg, layer_min_size, wb.bits, bucket_size, register_step,
                                      std::move(candidates), period, std::move(assignment), codec);
        },
        py::arg("reducer"), py::arg("backend"), py::arg("layer_min_size"), py::arg("bits"), py::arg("bucket_size"),
        py::arg("register_step") = 2, py::arg("candidates") = std::vector<int64_t>{}, py::arg("period") = 1,
        py::arg("assignment") = Assignment{});
  m.def("layer_wire_bytes", &layer_wire_bytes, py::arg("numel"), py::arg("bits"), py::arg("bucket_size"));
  m.def("allocate_bits",
        [](py::array_t<double, py::array::c_style | py::array::forcecast> errors, const std::vector<int64_t>& numels,
           const std::vector<int64_t>& bucket_sizes, const std::vector<int>& candidates, int64_t budget_bytes,
           const std::optional<std::vector<int>>& current, int64_t resolution, std::optional<int> target_bits) {
          const int64_t L = (int64_t)numels.size(), K = (int64_t)candidates.size();
          TORCH_CHECK(errors.ndim() == 2 && errors.shape(0) == L && errors.shape(1) == K,
                      "allocate_bits: errors must be [", L, ", ", K, "]");
          TORCH_CHECK(K >= 1 && resolution >= 1 && (int64_t)bucket_sizes.size() >= L,
                      "allocate_bits: need a candidate, resolution >= 1 and a bucket size per layer");
          py::gil_scoped_release nogil;
          return allocate_bits(errors.data(), L, numels, bucket_sizes, candidates, budget_bytes,
                               current ? &*current : nullptr, resolution, target_bits);
        },
        py::arg("errors"), py::arg("numels"), py::arg("bucket_sizes"), py::arg("candidates"), py::arg("budget_bytes"),
        py::arg("current") = py::none(), py::arg("resolution") = 4096, py::arg("target_bits") = py::none());

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
        py::arg("seed") = 0, py::arg("seq") = 0, py::arg("min_lane_elems") = 2048, py::arg("prescale") = py::none(),
        py::arg("bits") = py::none());
  m.def("reduce_scatter_simulate", &py_reduce_scatter_simulate, py::arg("inputs"), py::arg("outputs"),
        py::arg("shard_layers"), py::arg("lanes") = 1, py::arg("average") = false, py::arg("skip_incomplete") = false,
        py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0, py::arg("min_lane_elems") = 2048,
        py::arg("prescale") = py::none(), py::arg("bits") = py::none());
  m.def("all_to_all_simulate", &py_all_to_all_simulate, py::arg("inputs"), py::arg("outputs"), py::arg("counts"),
        py::arg("bits") = 8, py::arg("bucket_size") = 512, py::arg("stochastic") = false, py::arg("seed") = 0,
        py::arg("seq") = 0, py::arg("output_scales") = py::none());
  m.def(
      "a2a_bits",
      [](const A2aBitsArg& bits, bool stochastic, const std::string& op) {
        const A2aBits wb = a2a_bits(bits, stochastic, op.c_str());
        return std::make_tuple(wb.bits, (int)wb.codec);
      },
      py::arg("bits"), py::arg("stochastic") = false, py::arg("op") = "all_to_all");
  m.def("a2a_rng_stream", [](int src, int dst) { return (int64_t)a2a_rng_stream(src, dst); }, py::arg("src"),
        py::arg("dst"));
  // The 16 random bits of n consecutive elements from first_elem on, as the stochastic encoders draw
  // them: element i takes half i % 8 of rounding_bits of the group at first_elem + 8 * (i / 8). The
  // stream is the raw word (rank * 2 + phase, or a2a_rng_stream). For the references of the SR codecs.
  m.def(
      "philox_u16",
      [](uint64_t seed, uint32_t seq, uint32_t stream, uint32_t first_elem, int64_t n) {
        TORCH_CHECK(n >= 0, "philox_u16: n must be >= 0");
        RngKey k{(uint32_t)seed, (uint32_t)(seed >> 32), seq, stream, 1u};
        at::Tensor out = at::empty({n}, at::kInt);
        int32_t* o = out.data_ptr<int32_t>();
        for (int64_t g = 0; g < n; g += 8) {
          const Philox4 a = rounding_bits(k, first_elem + (uint32_t)g);
          for (int64_t j = 0; j < 8 && g + j < n; ++j) o[g + j] = (int32_t)((a.v[j >> 1] >> ((j & 1) * 16)) & 0xFFFFu);
        }
        return out;
      },
      py::arg("seed"), py::arg("seq"), py::arg("stream"), py::arg("first_elem"), py::arg("n"));
  m.attr("A2A_MAX_WORLD") = (int64_t)kA2aMaxWorld;
  m.def("a2a_remote_wire", &py_a2a_remote_wire, py::arg("counts"), py::arg("rank"), py::arg("local_size"),
        py::arg("bits"), py::arg("bucket_size"), py::arg("dtype") = 0);
  m.def("a2a_pack", &py_a2a_pack, py::arg("input"), py::arg("counts"), py::arg("rank"), py::arg("local_size"),
        py::arg("bits"), py::arg("bucket_size"), py::arg("stochastic") = false, py::arg("seed") = 0,
        py::arg("seq") = 0, py::arg("out") = py::none());
  m.def("a2a_unpack", &py_a2a_unpack, py::arg("records"), py::arg("output"), py::arg("counts"), py::arg("rank"),
        py::arg("local_size"), py::arg("bits"), py::arg("bucket_size"), py::arg("output_scales") = py::none());
  m.def("a2a_items", &py_a2a_items, py::arg("numel"), py::arg("bits"), py::arg("bucket_size"), py::arg("dtype") = 0);
  m.def(
      "a2a_rows_fit",
      [](int64_t row, int bits, int64_t bucket, int dtype) {
        return row >= 1 && row < (1ll << 32) && a2a_rows_fit((uint32_t)row, bits, (uint32_t)bucket, dtype_size(dtype));
      },
      py::arg("row"), py::arg("bits"), py::arg("bucket_size"), py::arg("dtype") = 0);
  m.def("a2a_windows", &py_a2a_windows, py::arg("numel"), py::arg("bits"), py::arg("bucket_size"), py::arg("dtype"),
        py::arg("slot_bytes"), py::arg("lanes"));
  m.def("all_gather_simulate", &py_all_gather_simulate, py::arg("inputs"), py::arg("outputs"),
        py::arg("shard_layers"), py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0,
        py::arg("bits") = py::none(), py::arg("output_scales") = py::none());
  m.def("oneshot_simulate", &py_oneshot_simulate, py::arg("tensors"), py::arg("layers"), py::arg("lanes") = 1,
        py::arg("average") = false, py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
        py::arg("seed") = 0, py::arg("seq") = 0, py::arg("min_lane_elems") = 2048, py::arg("prescale") = py::none(),
        py::arg("bits") = py::none());
  m.def("quantize", &py_quantize, py::arg("tensor"), py::arg("layers"), py::arg("world") = 1, py::arg("lanes") = 1,
        py::arg("skip_incomplete") = false, py::arg("prescale") = 1.0f, py::arg("stochastic") = false,
        py::arg("seed") = 0, py::arg("seq") = 0, py::arg("rank") = 0, py::arg("phase") = 0,
        py::arg("min_lane_elems") = 2048);
  m.def("dequantize", &py_dequantize, py::arg("wire"), py::arg("like"), py::arg("layers"), py::arg("world") = 1,
        py::arg("lanes") = 1, py::arg("skip_incomplete") = false, py::arg("min_lane_elems") = 2048);

  // The gate gradient of the weighted top-k combine (combine_gate_grad_kernel, DESIGN §2.13e) on the
  // current stream: grad_out [T, ...] and slots [T * k, ...] contiguous, of one dtype, any alignment;
  // returns grad_gate [T, k] float32.
  m.def(
      "combine_gate_grad",
      [](const at::Tensor& grad_out, const at::Tensor& slots, int64_t k) {
        TORCH_CHECK_VALUE(k >= 1 && k <= 32, "combine_gate_grad: k = ", k, " is not in 1..32");
        TORCH_CHECK_VALUE(grad_out.is_cuda() && slots.is_cuda() && grad_out.device() == slots.device() &&
                              grad_out.is_contiguous() && slots.is_contiguous() && grad_out.dim() >= 1 &&
                              slots.scalar_type() == grad_out.scalar_type(),
                          "combine_gate_grad: contiguous CUDA float32, float16 or bfloat16 tensors of one dtype");
        const int64_t T = grad_out.size(0), H = T > 0 ? grad_out.numel() / T : 0;
        TORCH_CHECK_VALUE(slots.numel() == T * k * H && H < (1ll << 32), "combine_gate_grad: slots must hold T * k = ",
                          T * k, " rows of the ", H, " elements of a grad_out row");
        c10::cuda::CUDAGuard g(grad_out.device());
        at::Tensor out = at::empty({T, k}, grad_out.options().dtype(at::kFloat));
        cuda_check(launch_combine_gate_grad(grad_out.data_ptr(), slots.data_ptr(), out.data_ptr<float>(),
                                            cgx_dtype(grad_out), (uint64_t)T, (uint32_t)k, (uint32_t)H,
                                            c10::cuda::getCurrentCUDAStream()),
                   "launch_combine_gate_grad");
        return out;
      },
      py::arg("grad_out"), py::arg("slots"), py::arg("k"));

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
        py::arg("stochastic") = false, py::arg("prescale") = 1.0, py::arg("skip_incomplete") = false,
        py::arg("chunks") = 1, py::arg("skip_chunk") = -1);
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
           py::arg("seq") = 0, py::arg("bits") = py::none())
      .def("allreduce_oneshot", &LocalSraGroup::allreduce_oneshot, py::arg("tensors"), py::arg("layers"),
           py::arg("average") = false, py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
           py::arg("seed") = 0, py::arg("seq") = 0, py::arg("bits") = py::none())
      .def("reduce_scatter", &LocalSraGroup::reduce_scatter, py::arg("inputs"), py::arg("outputs"),
           py::arg("shard_layers"), py::arg("average") = false, py::arg("skip_incomplete") = false,
           py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0, py::arg("bits") = py::none())
      .def("all_gather", &LocalSraGroup::all_gather, py::arg("inputs"), py::arg("outputs"), py::arg("shard_layers"),
           py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0, py::arg("bits") = py::none(),
           py::arg("output_scales") = py::none())
      .def("all_to_all", &LocalSraGroup::all_to_all, py::arg("inputs"), py::arg("outputs"), py::arg("counts"),
           py::arg("bits") = 8, py::arg("bucket_size") = 512, py::arg("stochastic") = false, py::arg("seed") = 0,
           py::arg("seq") = 0, py::arg("input_index") = IndexList{}, py::arg("output_index") = IndexList{},
           py::arg("row") = 1, py::arg("output_scales") = py::none(), py::arg("gate") = IndexList{},
           py::arg("combine_out") = IndexList{}, py::arg("input_scale") = IndexList{})
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
           py::arg("seed") = 0, py::arg("seq") = 0, py::arg("prescale") = py::none(), py::arg("bits") = py::none())
      .def("broadcast_compressed", &LocalReducerGroup::broadcast_compressed, py::arg("tensors"), py::arg("layers"),
           py::arg("root"), py::arg("skip_incomplete") = false, py::arg("stochastic") = false, py::arg("seed") = 0,
           py::arg("seq") = 0, py::arg("bits") = py::none())
      .def("reduce_scatter", &LocalReducerGroup::reduce_scatter, py::arg("inputs"), py::arg("outputs"),
           py::arg("shard_layers"), py::arg("average") = false, py::arg("skip_incomplete") = false,
           py::arg("stochastic") = false, py::arg("seed") = 0, py::arg("seq") = 0, py::arg("prescale") = py::none(),
           py::arg("bits") = py::none())
      .def("all_to_all", &LocalReducerGroup::all_to_all, py::arg("inputs"), py::arg("outputs"), py::arg("counts"),
           py::arg("bits") = 8, py::arg("bucket_size") = 512, py::arg("stochastic") = false, py::arg("seed") = 0,
           py::arg("seq") = 0, py::arg("output_scales") = py::none(), py::arg("output_index") = IndexList{},
           py::arg("row") = 1, py::arg("gate") = IndexList{}, py::arg("combine_out") = IndexList{},
           py::arg("input_index") = IndexList{})
      .def("all_gather", &LocalReducerGroup::all_gather, py::arg("inputs"), py::arg("outputs"),
           py::arg("shard_layers"), py::arg("skip_incomplete") = false, py::arg("stochastic") = false,
           py::arg("seed") = 0, py::arg("seq") = 0, py::arg("bits") = py::none(), py::arg("output_scales") = py::none())
      .def("bytes_sent", &LocalReducerGroup::bytes_sent)
      .def("num_plans", &LocalReducerGroup::num_plans, py::arg("rank"))
      .def("plan_uploads", &LocalReducerGroup::plan_uploads, py::arg("rank"))
      .def("set_recording", &LocalReducerGroup::set_recording, py::arg("on"))
      .def("messages", &LocalReducerGroup::messages);
  py::class_<LocalEngineGroup>(m, "LocalEngineGroup")
      .def(py::init<int, int, const py::dict&, int, int64_t, int64_t>(), py::arg("world"), py::arg("local_size"),
           py::arg("config"), py::arg("lanes") = 2, py::arg("slot_bytes") = 1 << 20, py::arg("timeout_ms") = 20000)
      .def("allreduce", &LocalEngineGroup::allreduce, py::arg("tensors"), py::arg("average") = false,
           py::arg("explicit_bucket") = -1, py::arg("overlapped") = false, py::arg("bits") = py::none())
      .def("allreduce_layers", &LocalEngineGroup::allreduce_layers, py::arg("tensors"), py::arg("layers"),
           py::arg("average") = false, py::arg("bits") = py::none())
      .def("reduce_scatter",
           [](LocalEngineGroup& g, std::vector<at::Tensor> in, std::vector<at::Tensor> out, bool average,
              std::optional<std::vector<LayerTuple>> shard_layers, std::optional<A2aBitsArg> bits) {
             g.sharded(true, std::move(in), std::move(out), average, shard_layers, bits);
           },
           py::arg("inputs"), py::arg("outputs"), py::arg("average") = false, py::arg("shard_layers") = py::none(),
           py::arg("bits") = py::none())
      .def("all_gather",
           [](LocalEngineGroup& g, std::vector<at::Tensor> in, std::vector<at::Tensor> out,
              std::optional<std::vector<LayerTuple>> shard_layers, std::optional<A2aBitsArg> bits,
              std::optional<std::vector<at::Tensor>> output_scales) {
             g.sharded(false, std::move(in), std::move(out), false, shard_layers, bits, output_scales);
           },
           py::arg("inputs"), py::arg("outputs"), py::arg("shard_layers") = py::none(), py::arg("bits") = py::none(),
           py::arg("output_scales") = py::none())
      .def("all_to_all", &LocalEngineGroup::all_to_all, py::arg("inputs"), py::arg("outputs"), py::arg("counts"),
           py::arg("bits") = 8, py::arg("bucket_size") = 512, py::arg("stochastic") = false, py::arg("seed") = 0,
           py::arg("output_scales") = py::none(), py::arg("input_index") = IndexList{},
           py::arg("output_index") = IndexList{}, py::arg("input_scale") = IndexList{}, py::arg("gate") = IndexList{},
           py::arg("combine_out") = IndexList{}, py::arg("row") = 1)
      .def("stats", &LocalEngineGroup::stats, py::arg("rank"))
      .def("check", &LocalEngineGroup::check)
      .def("log", &LocalEngineGroup::log, py::arg("rank"))
      .def("slot_bytes", &LocalEngineGroup::slot_bytes)
      .def("num_plans", &LocalEngineGroup::num_plans, py::arg("rank"));

  m.attr("MAX_BLOCK_ELEMS") = (int64_t)kMaxBlockElems;
  m.attr("MAX_PEERS") = (int64_t)kMaxPeers;
  m.attr("RAW_BITS") = (int64_t)kRawBits;
}

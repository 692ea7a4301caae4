#include "block_backend.h"

#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "../comm/symmetric_heap.h"
#include "../common/block_ops.h"
#include "../kernels/launch.h"

namespace cgx {
namespace {

// what the FP8 codecs of the block primitives support: compressed blocks of 8-bit plans, rounded to
// nearest unless the codec rounds stochastically (the reducers pass raw blocks with kMaxMin)
void check_fp8(const Plan& p, uint32_t first, uint32_t count, const RngKey& rng, WireCodec codec) {
  bool ok = p.uniform_bits == 8 && (!rng.enabled || fp8_sr(codec));
  for (uint32_t b = first; ok && b < first + count; ++b) ok = block_bits(p.blocks[b]) < kRawBits;
  if (!ok)
    throw std::invalid_argument("cgx: an FP8 codec needs compressed blocks of an 8-bit plan and round to nearest");
}

class CpuBackend : public BlockBackend {
 public:
  bool is_cuda() const override { return false; }
  void* alloc(size_t bytes) override {
    void* p = std::calloc(bytes ? bytes : 1, 1);
    if (!p) throw std::bad_alloc();
    return p;
  }
  void release(void* p) override { std::free(p); }
  void quantize(const DevicePlan& dp, const void* src, uint32_t first, uint32_t count, uint8_t* wire, float prescale,
                const RngKey& rng, cudaStream_t, WireCodec codec) override {
    const Plan& p = dp.plan;
    if (codec != kMaxMin) check_fp8(p, first, count, rng, codec);
    std::vector<float> acc(kMaxBlockElems);
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = p.blocks[b];
      cpu::load_block(src, p.dtype, d, prescale, acc.data());
      if (codec != kMaxMin)
        cpu::quantize_block_fp8(acc.data(), d, wire + d.wire_off, codec, rng);
      else
        cpu::quantize_block(acc.data(), p.dtype, d, wire + d.wire_off, rng, b);
    }
  }
  void accumulate(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, float* acc_f32,
                  uint32_t base_elem, const void* init_src, float prescale, cudaStream_t,
                  WireCodec codec) override {
    const Plan& p = dp.plan;
    if (codec != kMaxMin) check_fp8(p, first, count, RngKey{}, codec);
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = p.blocks[b];
      float* a = acc_f32 + (d.elem_off - base_elem);
      if (init_src) cpu::load_block(init_src, p.dtype, d, prescale, a);
      if (wire && codec != kMaxMin)
        cpu::decode_block_fp8_add(wire + d.wire_off, d, a, codec);
      else if (wire)
        cpu::decode_block_add(wire + d.wire_off, p.dtype, d, a);
    }
  }
  void quantize_f32(const DevicePlan& dp, const float* acc_f32, uint32_t base_elem, uint32_t first, uint32_t count,
                    uint8_t* wire, const RngKey& rng, void* out, cudaStream_t, WireCodec codec) override {
    const Plan& p = dp.plan;
    if (codec != kMaxMin) check_fp8(p, first, count, rng, codec);
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = p.blocks[b];
      if (codec != kMaxMin) {
        cpu::quantize_block_fp8(acc_f32 + (d.elem_off - base_elem), d, wire + d.wire_off, codec, rng);
        if (out) cpu::decode_block_fp8_store(wire + d.wire_off, p.dtype, d, out, codec);
        continue;
      }
      cpu::quantize_block(acc_f32 + (d.elem_off - base_elem), p.dtype, d, wire + d.wire_off, rng, b);
      if (out) cpu::decode_block_store(wire + d.wire_off, p.dtype, d, out);
    }
  }
  void dequantize(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, void* dst,
                  cudaStream_t, WireCodec codec) override {
    if (codec != kMaxMin) check_fp8(dp.plan, first, count, RngKey{}, codec);
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = dp.plan.blocks[b];
      if (codec != kMaxMin)
        cpu::decode_block_fp8_store(wire + d.wire_off, dp.plan.dtype, d, dst, codec);
      else
        cpu::decode_block_store(wire + d.wire_off, dp.plan.dtype, d, dst);
    }
  }
  void unpack_fp8(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, uint8_t* codes,
                  float* scales, cudaStream_t) override {
    check_fp8(dp.plan, first, count, RngKey{}, kE4M3);
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = dp.plan.blocks[b];
      cpu::unpack_block_fp8(wire + d.wire_off, d, codes, scales);
    }
  }
  void copy(void* dst, const void* src, size_t bytes, cudaStream_t) override { std::memcpy(dst, src, bytes); }
};

class CudaBackend : public BlockBackend {
 public:
  bool is_cuda() const override { return true; }
  void* alloc(size_t bytes) override {
    void* p = nullptr;
    cuda_check(cudaMalloc(&p, bytes ? bytes : 16), "cudaMalloc(reducer scratch)");
    cuda_check(cudaMemset(p, 0, bytes ? bytes : 16), "cudaMemset(reducer scratch)");
    // cudaMemset returns before it has run, on the legacy default stream, which does not order the
    // reducers' non-blocking streams: without this wait it can land after (and zero) the first kernel
    // writes to the buffer
    cuda_check(cudaStreamSynchronize(cudaStreamLegacy), "cudaMemset(reducer scratch): wait");
    return p;
  }
  void release(void* p) override { cudaFree(p); }
  void quantize(const DevicePlan& dp, const void* src, uint32_t first, uint32_t count, uint8_t* wire, float prescale,
                const RngKey& rng, cudaStream_t stream, WireCodec codec) override {
    if (codec != kMaxMin) check_fp8(dp.plan, first, count, rng, codec);
    cuda_check(launch_quantize_items(args(dp, first, count, codec), src, wire, prescale, rng, stream),
               "quantize_items");
  }
  void accumulate(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, float* acc_f32,
                  uint32_t base_elem, const void* init_src, float prescale, cudaStream_t stream,
                  WireCodec codec) override {
    if (codec != kMaxMin) check_fp8(dp.plan, first, count, RngKey{}, codec);
    cuda_check(launch_accumulate_items_f32(args(dp, first, count, codec), wire, acc_f32, base_elem, init_src, prescale,
                                           stream),
               "accumulate_items");
  }
  void quantize_f32(const DevicePlan& dp, const float* acc_f32, uint32_t base_elem, uint32_t first, uint32_t count,
                    uint8_t* wire, const RngKey& rng, void* out, cudaStream_t stream, WireCodec codec) override {
    if (codec != kMaxMin) check_fp8(dp.plan, first, count, rng, codec);
    cuda_check(launch_quantize_items_f32(args(dp, first, count, codec), acc_f32, base_elem, wire, rng, out, stream),
               "quantize_items_f32");
  }
  void dequantize(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, void* dst,
                  cudaStream_t stream, WireCodec codec) override {
    if (codec != kMaxMin) check_fp8(dp.plan, first, count, RngKey{}, codec);
    cuda_check(launch_dequantize_items(args(dp, first, count, codec), wire, dst, stream), "dequantize_items");
  }
  void unpack_fp8(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, uint8_t* codes,
                  float* scales, cudaStream_t stream) override {
    check_fp8(dp.plan, first, count, RngKey{}, kE4M3);
    if (count == 0) return;
    cuda_check(launch_unpack_items_fp8(args(dp, first, count), wire, codes, scales, dp.plan.blocks[first].bucket, stream),
               "unpack_items_fp8");
  }
  void copy(void* dst, const void* src, size_t bytes, cudaStream_t stream) override {
    cuda_check(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, stream), "cudaMemcpyAsync");
  }

 private:
  // blocks [first, first+count) -> their warp items (items are emitted block by block)
  static ItemKernelArgs args(const DevicePlan& dp, uint32_t first, uint32_t count, WireCodec codec = kMaxMin) {
    ItemKernelArgs a;
    a.codec = codec;
    a.items = dp.d_items;
    a.first = dp.plan.block_item_first[first];
    a.count = dp.plan.block_item_first[first + count] - a.first;
    a.dtype = dp.plan.dtype;
    a.slice_elems = (int)dp.plan.slice_elems;
    a.uniform_bits = dp.plan.uniform_bits;
    if (a.count && !dp.d_items) throw std::logic_error("cgx: the device backend got a plan that was not uploaded");
    return a;
  }
};

}  // namespace

std::unique_ptr<BlockBackend> make_cpu_block_backend() { return std::make_unique<CpuBackend>(); }
std::unique_ptr<BlockBackend> make_cuda_block_backend() { return std::make_unique<CudaBackend>(); }

}  // namespace cgx

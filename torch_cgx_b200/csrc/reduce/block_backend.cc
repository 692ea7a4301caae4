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

class CpuBackend : public BlockBackend {
 public:
  bool is_cuda() const override { return false; }
  void* alloc(size_t bytes) override {
    void* p = std::calloc(bytes ? bytes : 1, 1);
    if (!p) throw std::bad_alloc();
    return p;
  }
  void release(void* p) override { std::free(p); }
  void bind(const Plan& plan, cudaStream_t) override { plan_ = &plan; }
  void quantize(const void* src, uint32_t first, uint32_t count, uint8_t* wire, float prescale, const RngKey& rng,
                cudaStream_t) override {
    std::vector<float> acc(kMaxBlockElems);
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = plan_->blocks[b];
      cpu::load_block(src, plan_->dtype, d, prescale, acc.data());
      cpu::quantize_block(acc.data(), plan_->dtype, d, wire + d.wire_off, rng, b);
    }
  }
  void accumulate(const uint8_t* wire, uint32_t first, uint32_t count, float* acc_f32, uint32_t base_elem,
                  const void* init_src, float prescale, cudaStream_t) override {
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = plan_->blocks[b];
      float* a = acc_f32 + (d.elem_off - base_elem);
      if (init_src) cpu::load_block(init_src, plan_->dtype, d, prescale, a);
      if (wire) cpu::decode_block_add(wire + d.wire_off, plan_->dtype, d, a);
    }
  }
  void quantize_f32(const float* acc_f32, uint32_t base_elem, uint32_t first, uint32_t count, uint8_t* wire,
                    const RngKey& rng, void* out, cudaStream_t) override {
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = plan_->blocks[b];
      cpu::quantize_block(acc_f32 + (d.elem_off - base_elem), plan_->dtype, d, wire + d.wire_off, rng, b);
      if (out) cpu::decode_block_store(wire + d.wire_off, plan_->dtype, d, out);
    }
  }
  void dequantize(const uint8_t* wire, uint32_t first, uint32_t count, void* dst, cudaStream_t) override {
    for (uint32_t b = first; b < first + count; ++b) {
      const BlockDesc& d = plan_->blocks[b];
      cpu::decode_block_store(wire + d.wire_off, plan_->dtype, d, dst);
    }
  }
  void copy(void* dst, const void* src, size_t bytes, cudaStream_t) override { std::memcpy(dst, src, bytes); }

 private:
  const Plan* plan_ = nullptr;
};

class CudaBackend : public BlockBackend {
 public:
  ~CudaBackend() override {
    if (d_items_) cudaFree(d_items_);
  }
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
  void unbind() override { plan_ = nullptr; }
  void bind(const Plan& plan, cudaStream_t stream) override {
    if (plan_ == &plan) return;  // plans are cached by the reducers and immutable: upload once
    plan_ = &plan;
    const size_t bytes = plan.items.size() * sizeof(WarpItem);
    if (bytes > cap_) {
      if (d_items_) {
        cuda_check(cudaStreamSynchronize(stream), "sync before plan realloc");
        cudaFree(d_items_);
      }
      cuda_check(cudaMalloc((void**)&d_items_, bytes), "cudaMalloc(plan)");
      cap_ = bytes;
    }
    if (bytes)
      cuda_check(cudaMemcpyAsync(d_items_, plan.items.data(), bytes, cudaMemcpyHostToDevice, stream), "upload plan");
  }
  void quantize(const void* src, uint32_t first, uint32_t count, uint8_t* wire, float prescale, const RngKey& rng,
                cudaStream_t stream) override {
    cuda_check(launch_quantize_items(args(first, count), src, wire, prescale, rng, stream), "quantize_items");
  }
  void accumulate(const uint8_t* wire, uint32_t first, uint32_t count, float* acc_f32, uint32_t base_elem,
                  const void* init_src, float prescale, cudaStream_t stream) override {
    cuda_check(launch_accumulate_items_f32(args(first, count), wire, acc_f32, base_elem, init_src, prescale, stream),
               "accumulate_items");
  }
  void quantize_f32(const float* acc_f32, uint32_t base_elem, uint32_t first, uint32_t count, uint8_t* wire,
                    const RngKey& rng, void* out, cudaStream_t stream) override {
    cuda_check(launch_quantize_items_f32(args(first, count), acc_f32, base_elem, wire, rng, out, stream),
               "quantize_items_f32");
  }
  void dequantize(const uint8_t* wire, uint32_t first, uint32_t count, void* dst, cudaStream_t stream) override {
    cuda_check(launch_dequantize_items(args(first, count), wire, dst, stream), "dequantize_items");
  }
  void copy(void* dst, const void* src, size_t bytes, cudaStream_t stream) override {
    cuda_check(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, stream), "cudaMemcpyAsync");
  }

 private:
  // blocks [first, first+count) -> their warp items (items are emitted block by block)
  ItemKernelArgs args(uint32_t first, uint32_t count) const {
    ItemKernelArgs a;
    a.items = d_items_;
    a.first = plan_->block_item_first[first];
    a.count = plan_->block_item_first[first + count] - a.first;
    a.dtype = plan_->dtype;
    a.slice_elems = (int)plan_->slice_elems;
    a.uniform_bits = plan_->uniform_bits;
    return a;
  }
  const Plan* plan_ = nullptr;
  WarpItem* d_items_ = nullptr;
  size_t cap_ = 0;
};

}  // namespace

std::unique_ptr<BlockBackend> make_cpu_block_backend() { return std::make_unique<CpuBackend>(); }
std::unique_ptr<BlockBackend> make_cuda_block_backend() { return std::make_unique<CudaBackend>(); }

}  // namespace cgx

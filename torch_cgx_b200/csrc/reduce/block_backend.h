// Device abstraction for the generic reducers: the four block primitives on
// either host memory (common/block_ops.h) or device memory (kernels/quantize.cu).
// Reference role: Compressor::{Compress,Decompress,Add} over GPUContext
// (/root/reference/src/common/compressor.cc:62-220, gpu_context.h:67-100).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <memory>

#include "../common/philox.h"
#include "../common/plan.h"
#include "../common/quant_math.h"
#include "plan_cache.h"

namespace cgx {

class BlockBackend {
 public:
  virtual ~BlockBackend() = default;
  virtual bool is_cuda() const = 0;
  // scratch memory of the backend's kind (zero-initialised)
  virtual void* alloc(size_t bytes) = 0;
  virtual void release(void* p) = 0;
  // The block primitives work on blocks [first, first+count) of `dp`'s plan; the device backend
  // reads its uploaded tables (PlanCache::upload), the host backend the plan alone.
  // wire = quantize(src[T] * prescale). An FP8 `codec` (common/quant_math.h) needs compressed blocks
  // of an 8-bit plan and deterministic rounding; its records are read back by dequantize and
  // accumulate with the same codec.
  virtual void quantize(const DevicePlan& dp, const void* src, uint32_t first, uint32_t count, uint8_t* wire,
                        float prescale, const RngKey& rng, cudaStream_t stream, WireCodec codec = kMaxMin) = 0;
  // acc_f32[elem_off - base_elem + i] = float(init_src[elem_off + i]) * prescale   (init_src != nullptr)
  // acc_f32[...] += decode(wire)                                                   (wire != nullptr)
  // (an FP8 codec adds fl(float(code) * unit), a separate rounding)
  virtual void accumulate(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, float* acc_f32,
                          uint32_t base_elem, const void* init_src, float prescale, cudaStream_t stream,
                          WireCodec codec = kMaxMin) = 0;
  // wire = quantize(acc_f32); out[T] = decode(wire) when out != nullptr (an FP8 codec as in quantize)
  virtual void quantize_f32(const DevicePlan& dp, const float* acc_f32, uint32_t base_elem, uint32_t first,
                            uint32_t count, uint8_t* wire, const RngKey& rng, void* out, cudaStream_t stream,
                            WireCodec codec = kMaxMin) = 0;
  // dst[T] = decode(wire)
  virtual void dequantize(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, void* dst,
                          cudaStream_t stream, WireCodec codec = kMaxMin) = 0;
  // codes[elem_off + i] / scales[elem_off / bucket + b] = the undecoded FP8 codes and units of the
  // records (compressed blocks of an 8-bit plan whose bucket divides every block's offset)
  virtual void unpack_fp8(const DevicePlan& dp, const uint8_t* wire, uint32_t first, uint32_t count, uint8_t* codes,
                          float* scales, cudaStream_t stream) = 0;
  virtual void copy(void* dst, const void* src, size_t bytes, cudaStream_t stream) = 0;
};

std::unique_ptr<BlockBackend> make_cpu_block_backend();
std::unique_ptr<BlockBackend> make_cuda_block_backend();

}  // namespace cgx

#include "quant_error_table.h"

#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include <algorithm>
#include <cstring>

#include "../comm/symmetric_heap.h"
#include "../common/quant_error.h"
#include "../kernels/launch.h"

namespace cgx {

at::Tensor quantization_error_table(const at::Tensor& t, const std::vector<QErrSpan>& spans,
                                    const std::vector<int64_t>& candidates, bool stochastic, double prescale,
                                    bool skip_incomplete, int64_t chunks, int64_t skip_chunk) {
  TORCH_CHECK(t.device().is_cpu() || t.is_cuda(), "quantization_error: tensor must be on the CPU or a CUDA device");
  TORCH_CHECK(t.is_contiguous(), "quantization_error: tensor must be contiguous");
  TORCH_CHECK(chunks >= 1 && chunks <= (1 << 20), "quantization_error: chunks must be in 1..2^20, got ", chunks);
  TORCH_CHECK(t.numel() % chunks == 0, "quantization_error: ", t.numel(), " elements do not split into ", chunks,
              " chunks");
  TORCH_CHECK(skip_chunk >= -1 && skip_chunk < chunks, "quantization_error: skip_chunk ", skip_chunk,
              " is outside [-1, ", chunks, ")");
  const int64_t S = t.numel() / chunks;
  int dt = kF32;
  switch (t.scalar_type()) {
    case at::kFloat: dt = kF32; break;
    case at::kHalf: dt = kF16; break;
    case at::kBFloat16: dt = kBF16; break;
    default: TORCH_CHECK(false, "cgx: unsupported dtype ", t.scalar_type(), " (need float32/float16/bfloat16)");
  }
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
  ls.reserve(spans.size());
  for (const QErrSpan& s : spans) {
    const int64_t off = s.elem_off, n = s.numel, bucket = s.bucket;
    if (chunks == 1) {
      TORCH_CHECK(off >= 0 && n >= 0 && off + n <= t.numel(), "quantization_error: layer (", off, ", ", n,
                  ") is outside the tensor of ", t.numel(), " elements");
    } else {
      TORCH_CHECK(off >= 0 && n >= 0 && off + n <= S, "quantization_error: layer (", off, ", ", n,
                  ") reaches past the chunk of ", S, " elements");
    }
    TORCH_CHECK(bucket >= 1, "quantization_error: bucket size must be >= 1, got ", bucket);
    // clamped like the plan clamps it (plan.cc: push_segment)
    const uint32_t B = (uint32_t)std::min<int64_t>(bucket, kMaxBlockElems);
    // with skip_incomplete the tail bucket travels raw: no error
    ls.push_back({(uint64_t)off, skip_incomplete ? (uint64_t)n / B * B : (uint64_t)n, B, 0});
  }
  const int64_t L = (int64_t)ls.size();
  if (t.device().is_cpu()) {
    at::Tensor out = at::zeros({L, (int64_t)K}, at::kDouble);
    cpu::quantization_error(t.data_ptr(), dt, ls, bits, K, stochastic, (float)prescale, out.data_ptr<double>(),
                            (int)chunks, (uint64_t)S, (int)skip_chunk);
    return out;
  }
  c10::cuda::CUDAGuard g(t.device());
  auto stream = c10::cuda::getCurrentCUDAStream();
  const std::vector<uint64_t> first = qerr_first(ls);
  const uint64_t nb = first.back();
  const uint64_t total = nb * (uint64_t)(chunks - (skip_chunk >= 0 ? 1 : 0));
  TORCH_CHECK(total < (1ull << 34), "quantization_error: too many buckets for one launch");
  const size_t lbytes = ls.size() * sizeof(QErrLayer), fbytes = first.size() * sizeof(uint64_t);
  // layer table and first buckets go up in one copy from pinned memory: no synchronisation with the stream
  at::Tensor host = at::empty({(int64_t)(lbytes + fbytes)}, at::TensorOptions().dtype(at::kByte).pinned_memory(true));
  std::memcpy(host.data_ptr<uint8_t>(), ls.data(), lbytes);
  std::memcpy(host.data_ptr<uint8_t>() + lbytes, first.data(), fbytes);
  at::Tensor dev = at::empty({(int64_t)(lbytes + fbytes)}, t.options().dtype(at::kByte));
  dev.copy_(host, /*non_blocking=*/true);
  at::Tensor partial = at::empty({(int64_t)std::max<uint64_t>(1, total * (uint64_t)K)}, t.options().dtype(at::kFloat));
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
  a.chunks = (int)chunks;
  a.chunk_stride = (uint64_t)S;
  a.skip_chunk = (int)skip_chunk;
  cuda_check(launch_quantization_error(a, stream), "quantization_error");
  return out;
}

}  // namespace cgx

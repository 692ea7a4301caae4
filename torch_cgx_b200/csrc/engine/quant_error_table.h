// Per-layer quantization-error table of a flat gradient: the host side of
// `ops.quantization_error`, shared by its binding and by the adaptive native DDP hook.
#pragma once
#include <ATen/ATen.h>

#include <cstdint>
#include <vector>

namespace cgx {

struct QErrSpan {
  int64_t elem_off;
  int64_t numel;
  int64_t bucket;  // quantization bucket; clamped to kMaxBlockElems like the plan clamps it
};

// [spans.size(), candidates.size()] float64 on t.device(): the squared error one quantization round
// trip adds to every span at every candidate width (common/quant_error.h). CPU tensors run the C++
// path; CUDA tensors launch the sm_90a kernel on the current stream without synchronising. Checks
// its arguments and throws c10::Error on bad ones.
//
// chunks > 1 is the sharded mode of a reduce-scatter input: t holds `chunks` copies of the span
// table at stride t.numel() / chunks (the spans must fit in one chunk), and every row sums the error
// of its span over all chunks except skip_chunk (-1: none). chunks = 1 is the plain table.
at::Tensor quantization_error_table(const at::Tensor& t, const std::vector<QErrSpan>& spans,
                                    const std::vector<int64_t>& candidates, bool stochastic, double prescale,
                                    bool skip_incomplete, int64_t chunks = 1, int64_t skip_chunk = -1);

}  // namespace cgx

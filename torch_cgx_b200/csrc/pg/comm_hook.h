// Native DDP communication hook: the C++ twin of cgx_hook/CGXState
// (/root/reference/cgx_utils/allreduce_hooks.py:29-73). Registered straight on
// the c10d::Reducer, so the per-bucket path never enters Python: no GIL, no
// Python future callback -- in launch-bound regimes (small per-GPU batch) the
// Python hook costs ~50 us per bucket, which is visible against NCCL's built-in
// C++ allreduce hook.
//
// With candidate widths it is also the twin of AdaptiveCGXState.bucket_hook
// (parallel/adaptive.py): every `period` steps it estimates each compressed layer's
// quantization error before the bucket's allreduce, and at the first bucket of the next step
// it sums the estimates over the group, lets group rank 0 choose the widths
// (common/bit_allocation.h) and applies the widths rank 0 broadcast.
#pragma once
#include <torch/csrc/distributed/c10d/comm.hpp>
#include <torch/csrc/distributed/c10d/reducer.hpp>

#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <utility>
#include <vector>

#include "process_group_cgx.h"

namespace cgx {

struct AdaptedLayer {
  int64_t bucket, layer, elem_off, numel;  // elem_off: inside the bucket's flat buffer
};

struct HookState {
  c10::intrusive_ptr<ProcessGroupCGX> pg;
  int64_t layer_min_size = 1024;
  int bits = 32;
  int bucket_size = 1024;
  std::optional<WireCodec> codec;  // wire format of the 8-bit layers; none: CGX_COMPRESSION_FORMAT's
  int register_step = 2;  // DDP rebuilds its buckets after the first iteration
  std::atomic<int64_t> step{0};

  // ---- adaptive widths: off while `candidates` is empty ----
  std::vector<int64_t> candidates;
  int64_t period = 1;
  std::mutex mu;  // guards everything below: Python may read it while the hook runs
  std::map<int64_t, std::vector<AdaptedLayer>> by_bucket;  // compressed layers, registration
  std::map<int64_t, at::Tensor> tables;                    // bucket -> pending [layers, K] estimate
  std::map<std::pair<int64_t, int64_t>, int> assignment;   // (bucket, layer) -> applied width
  std::map<std::pair<int64_t, int64_t>, int> loaded;       // applied at registration
  at::Tensor last_errors;                                  // group-summed [rows, K], CPU; undefined before
  bool step_open = false;
  c10::Device device{c10::kCPU};

  bool adaptive() const { return !candidates.empty(); }
  // rows of every registered bucket, in bucket order (the rows of last_errors after a decision
  // that covered every bucket)
  std::vector<AdaptedLayer> adapted_layers();
};

class CgxCommHook : public c10d::CommHookInterface {
 public:
  explicit CgxCommHook(std::shared_ptr<HookState> st) : st_(std::move(st)) {}
  c10::intrusive_ptr<c10::ivalue::Future> runHook(c10d::GradBucket& bucket) override;
  at::Tensor parseHookResult(const c10::IValue& result) override {
    return c10d::detail::parseCppCommHookResult(result);
  }

 private:
  void register_bucket(HookState& s, c10d::GradBucket& bucket);
  void estimate(HookState& s, int64_t b, const at::Tensor& buf);
  void decide(HookState& s);
  std::shared_ptr<HookState> st_;
};

// registers the hook on `reducer` (a torch.distributed.Reducer) and returns the shared state.
// Non-empty `candidates` turns on adaptive widths; `loaded` is applied at registration. An FP8
// `codec` (bits 8, fixed widths) sends the compressed layers as FP8 codes.
std::shared_ptr<HookState> register_native_hook(const std::shared_ptr<c10d::Reducer>& reducer,
                                                c10::intrusive_ptr<ProcessGroupCGX> pg, int64_t layer_min_size,
                                                int bits, int bucket_size, int register_step,
                                                std::vector<int64_t> candidates = {}, int64_t period = 1,
                                                std::map<std::pair<int64_t, int64_t>, int> loaded = {},
                                                std::optional<WireCodec> codec = std::nullopt);

}  // namespace cgx

#include "comm_hook.h"

#include <c10/cuda/CUDAGraphsC10Utils.h>

#include "../common/bit_allocation.h"
#include "../common/config.h"
#include "../common/layers.h"
#include "../engine/quant_error_table.h"

namespace cgx {

namespace {

bool capturing(const at::Tensor& t) {
  return t.is_cuda() && c10::cuda::currentStreamCaptureStatusMayInitCtx() != c10::cuda::CaptureStatus::None;
}

}  // namespace

std::vector<AdaptedLayer> HookState::adapted_layers() {
  std::lock_guard<std::mutex> lk(mu);
  std::vector<AdaptedLayer> out;
  for (const auto& kv : by_bucket) out.insert(out.end(), kv.second.begin(), kv.second.end());
  return out;
}

c10::intrusive_ptr<c10::ivalue::Future> CgxCommHook::runHook(c10d::GradBucket& bucket) {
  HookState& s = *st_;
  const int64_t step = s.step.load(std::memory_order_relaxed);
  const size_t idx = bucket.getIndex();
  if (s.adaptive()) {
    std::lock_guard<std::mutex> lk(s.mu);
    if (!s.step_open) {
      s.step_open = true;
      if (!s.tables.empty()) {
        TORCH_CHECK(!capturing(bucket.getBufferRef()),
                    "cgx native hook: a decision step of adaptive widths cannot run during CUDA graph capture");
        decide(s);
      }
    }
    if (step == s.register_step) register_bucket(s, bucket);
    const bool adapt = s.bits <= 8 && step >= s.register_step;
    auto it = s.by_bucket.find((int64_t)idx);
    if (adapt && (step - s.register_step) % s.period == 0 && it != s.by_bucket.end() && !it->second.empty()) {
      TORCH_CHECK(!capturing(bucket.getBufferRef()),
                  "cgx native hook: an estimate step of adaptive widths cannot run during CUDA graph capture");
      estimate(s, (int64_t)idx, bucket.getBufferRef());
    }
    if (bucket.isLast()) s.step_open = false;
  } else if (step == s.register_step) {
    register_bucket(s, bucket);
  }
  const bool registered = step >= s.register_step;
  if (bucket.isLast()) s.step.fetch_add(1, std::memory_order_relaxed);
  // average == true: the 1/world scale is applied inside the kernel, before quantization
  auto work = s.pg->allreduce_bucket(bucket.getBufferRef(), registered ? (int64_t)idx : -1, true, s.codec);
  return work->getFuture();
}

void CgxCommHook::register_bucket(HookState& s, c10d::GradBucket& bucket) {
  // tell the backend the layer structure of this bucket: 1-D / small layers stay uncompressed
  const int64_t b = (int64_t)bucket.getIndex();
  const std::vector<at::Tensor> grads = bucket.getGradients();
  std::vector<AdaptedLayer> mine;
  int64_t off = 0;
  for (size_t i = 0; i < grads.size(); ++i) {
    const at::Tensor& g = grads[i];
    const bool compress = g.dim() > 1 && g.numel() >= s.layer_min_size;
    LayerRegistry::instance().register_layer((unsigned)b, (unsigned)i, g.numel(), compress ? s.bits : kRawBits,
                                             s.bucket_size);
    if (compress && s.bits <= 8) mine.push_back({b, (int64_t)i, off, g.numel()});
    off += g.numel();
  }
  if (!s.adaptive()) return;
  s.by_bucket[b] = mine;
  for (const AdaptedLayer& l : mine) {
    auto it = s.loaded.find({b, l.layer});
    if (it == s.loaded.end()) continue;
    LayerRegistry::instance().set_bits((unsigned)b, (unsigned)l.layer, it->second);
    s.assignment[{b, l.layer}] = it->second;
  }
}

void CgxCommHook::estimate(HookState& s, int64_t b, const at::Tensor& buf) {
  const CompressionEnv env = CompressionEnv::read();
  std::vector<QErrSpan> spans;
  for (const AdaptedLayer& l : s.by_bucket[b]) spans.push_back({l.elem_off, l.numel, (int64_t)s.bucket_size});
  s.device = buf.device();
  // enqueued before the in-place allreduce, on the same stream: no synchronisation
  s.tables[b] = quantization_error_table(buf, spans, s.candidates, env.stochastic, 1.0 / s.pg->getSize(),
                                         env.skip_incomplete);
}

void CgxCommHook::decide(HookState& s) {
  const int64_t K = (int64_t)s.candidates.size();
  std::vector<at::Tensor> flat;
  std::vector<AdaptedLayer> rows;
  for (const auto& kv : s.tables) {
    flat.push_back(kv.second.reshape({-1}));
    const std::vector<AdaptedLayer>& ls = s.by_bucket[kv.first];
    rows.insert(rows.end(), ls.begin(), ls.end());
  }
  s.tables.clear();
  // float64 never takes the compressed path: the group's delegate sums it
  std::vector<at::Tensor> sum{at::cat(flat)};
  s.pg->allreduce(sum)->wait();
  const at::Tensor table = sum[0].view({-1, K}).cpu();
  TORCH_CHECK(table.size(0) == (int64_t)rows.size(), "cgx native hook: error table has ", table.size(0),
              " rows for ", rows.size(), " adapted layers");
  at::Tensor choice = at::zeros({(int64_t)rows.size()}, at::kInt);
  if (s.pg->getRank() == 0) {
    const int64_t L = (int64_t)rows.size();
    std::vector<int64_t> numels(L), buckets(L, s.bucket_size);
    std::vector<int> current(L), cands(s.candidates.begin(), s.candidates.end());
    int64_t budget = 0;
    for (int64_t i = 0; i < L; ++i) {
      numels[i] = rows[i].numel;
      budget += layer_wire_bytes(rows[i].numel, s.bits, s.bucket_size);
      auto it = s.assignment.find({rows[i].bucket, rows[i].layer});
      current[i] = it == s.assignment.end() ? s.bits : it->second;
    }
    const std::vector<int> picked = allocate_bits(table.contiguous().data_ptr<double>(), L, numels, buckets, cands,
                                                  budget, &current, 4096, s.bits);
    std::copy(picked.begin(), picked.begin() + L, choice.data_ptr<int32_t>());
  }
  std::vector<at::Tensor> bc{choice.to(s.device)};
  c10d::BroadcastOptions o;
  o.rootRank = 0;
  s.pg->broadcast(bc, o)->wait();
  const at::Tensor widths = bc[0].cpu();
  const int32_t* w = widths.data_ptr<int32_t>();
  for (size_t i = 0; i < rows.size(); ++i) {
    LayerRegistry::instance().set_bits((unsigned)rows[i].bucket, (unsigned)rows[i].layer, w[i]);
    s.assignment[{rows[i].bucket, rows[i].layer}] = w[i];
  }
  s.last_errors = table;
}

std::shared_ptr<HookState> register_native_hook(const std::shared_ptr<c10d::Reducer>& reducer,
                                                c10::intrusive_ptr<ProcessGroupCGX> pg, int64_t layer_min_size,
                                                int bits, int bucket_size, int register_step,
                                                std::vector<int64_t> candidates, int64_t period,
                                                std::map<std::pair<int64_t, int64_t>, int> loaded,
                                                std::optional<WireCodec> codec) {
  TORCH_CHECK(period >= 1, "register_native_hook: period must be >= 1, got ", period);
  if (codec && *codec != kMaxMin) {
    if (!candidates.empty())
      throw std::invalid_argument("register_native_hook: adaptive widths have no FP8 formats");
    if (bits != 8) throw std::invalid_argument("register_native_hook: an FP8 format uses bits 8");
  }
  for (int64_t c : candidates)
    TORCH_CHECK(c >= 1 && c <= 8, "register_native_hook: candidate width ", c, " is outside 1..8");
  auto st = std::make_shared<HookState>();
  st->pg = std::move(pg);
  st->layer_min_size = layer_min_size;
  st->bits = bits;
  st->bucket_size = bucket_size;
  st->register_step = register_step;
  st->candidates = std::move(candidates);
  st->period = period;
  st->loaded = std::move(loaded);
  st->codec = codec;
  reducer->register_comm_hook(std::make_unique<CgxCommHook>(st));
  return st;
}

}  // namespace cgx

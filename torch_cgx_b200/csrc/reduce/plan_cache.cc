#include "plan_cache.h"

#include <algorithm>
#include <cstring>

#include "../comm/symmetric_heap.h"  // cuda_check
#include "../common/config.h"

namespace cgx {
namespace {

constexpr size_t kTableAlign = 256;
constexpr size_t kFirstBlockBytes = 1 << 20;

size_t align_table(size_t bytes) { return (bytes + kTableAlign - 1) / kTableAlign * kTableAlign; }
size_t items_bytes(const Plan& p) { return p.items.size() * sizeof(WarpItem); }
// both tables of a plan, items first, as placed in the arena
size_t table_bytes(const Plan& p) { return align_table(items_bytes(p)) + p.item_first.size() * sizeof(uint32_t); }

}  // namespace

PlanCache::PlanCache(size_t max_plans, size_t max_table_bytes)
    : max_plans_(max_plans), max_table_bytes_(max_table_bytes) {}

PlanCache::~PlanCache() {
  for (void* b : blocks_) cudaFree(b);
}

const DevicePlan& PlanCache::get(const std::vector<LayerSpec>& layers, const PlanOptions& opt, cudaStream_t stream) {
  const uint64_t key = plan_key(layers, opt);
  auto it = plans_.find(key);
  if (it != plans_.end()) return *it->second;
  auto dp = std::make_unique<DevicePlan>();
  dp->plan = build_plan(layers, opt);
  bool mc = true;
  for (const BlockDesc& bd : dp->plan.blocks) {
    const int bb = block_bits(bd);
    mc = mc && (block_is_raw(bd) || bb == 2 || bb == 4 || bb == 8);
  }
  dp->multicast_ok = mc;
  const size_t bytes = table_bytes(dp->plan);
  // workloads with ever-changing message sizes: drop everything rather than track the use of entries
  if (!plans_.empty() &&
      (plans_.size() >= max_plans_ || (max_table_bytes_ && table_bytes_ + bytes > max_table_bytes_)))
    drop(stream);
  if (log_level() >= 2) log_msg(2, "cgx: new plan %s", describe_plan(dp->plan).c_str());
  table_bytes_ += bytes;
  return *plans_.emplace(key, std::move(dp)).first->second;
}

void PlanCache::upload(const DevicePlan& entry, cudaStream_t stream) {
  if (entry.d_items || entry.plan.items.empty()) return;
  DevicePlan& dp = const_cast<DevicePlan&>(entry);  // owned (non-const) by plans_
  const Plan& p = dp.plan;
  // one copy per plan: both tables staged back to back as they are placed
  std::vector<uint8_t> host(table_bytes(p));
  std::memcpy(host.data(), p.items.data(), items_bytes(p));
  std::memcpy(host.data() + align_table(items_bytes(p)), p.item_first.data(), p.item_first.size() * sizeof(uint32_t));
  uint8_t* d = place(host.size());
  // pageable source: the runtime stages it before returning, so `host` may go
  cuda_check(cudaMemcpyAsync(d, host.data(), host.size(), cudaMemcpyHostToDevice, stream), "upload plan tables");
  dp.d_items = reinterpret_cast<WarpItem*>(d);
  dp.d_item_first = reinterpret_cast<uint32_t*>(d + align_table(items_bytes(p)));
  ++uploads_;
}

void PlanCache::drop(cudaStream_t stream) {
  // host-memory caches never uploaded anything, so there is nothing on the device to wait for
  if (!blocks_.empty()) cuda_check(cudaStreamSynchronize(stream), "sync before dropping the plan cache");
  for (void* b : blocks_) cudaFree(b);
  blocks_.clear();
  block_cap_ = block_used_ = 0;
  plans_.clear();
  table_bytes_ = 0;
  ++generation_;
}

uint8_t* PlanCache::place(size_t bytes) {
  bytes = align_table(bytes);
  if (blocks_.empty() || block_used_ + bytes > block_cap_) {
    // a new block, at least twice the last: the tables already placed keep their addresses
    block_cap_ = std::max(bytes, blocks_.empty() ? kFirstBlockBytes : 2 * block_cap_);
    void* b = nullptr;
    cuda_check(cudaMalloc(&b, block_cap_), "cudaMalloc(plan tables)");
    blocks_.push_back(b);
    block_used_ = 0;
  }
  uint8_t* p = static_cast<uint8_t*>(blocks_.back()) + block_used_;
  block_used_ += bytes;
  return p;
}

}  // namespace cgx

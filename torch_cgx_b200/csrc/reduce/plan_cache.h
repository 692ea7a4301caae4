// The one owner of plans and their device tables, for the fused kernels (FusedSra), the generic
// reducers (Reducer) and the pre-planned codec of the Python API.
//
// A plan is built on the first request for its (layers, options) key and kept until the cache is
// dropped as a whole. Its warp-item tables are copied to the device on the first upload() only, so
// a plan that never runs on the device (too large for the heap slots, or a host-memory reducer's)
// is never uploaded. The tables live back to back in device blocks owned by the cache; a full block
// is followed by a larger one, and nothing is freed before a drop or the cache's destruction, so a
// table's address stays valid as long as its entry.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <memory>
#include <unordered_map>
#include <vector>

#include "../common/plan.h"

namespace cgx {

struct DevicePlan {
  Plan plan;
  WarpItem* d_items = nullptr;       // flattened warp work list (device; null until uploaded)
  uint32_t* d_item_first = nullptr;  // [world * lanes + 1]
  bool multicast_ok = false;         // every compressed item has a width multimem.st can carry (2/4/8)
};

class PlanCache {
 public:
  // max_table_bytes = 0: no bound on the tables' bytes
  explicit PlanCache(size_t max_plans, size_t max_table_bytes = 0);
  ~PlanCache();
  PlanCache(const PlanCache&) = delete;
  PlanCache& operator=(const PlanCache&) = delete;

  // The plan of `layers` under `opt`, built on a miss. When inserting it would exceed max_plans or
  // max_table_bytes, every entry is dropped first: `stream` is synchronised (kernels still reading
  // the old tables finish before they are freed), the arena is released and generation() bumped.
  // A reference returned earlier is invalid after a later get() that dropped.
  const DevicePlan& get(const std::vector<LayerSpec>& layers, const PlanOptions& opt, cudaStream_t stream);
  // makes the tables of `dp` (an entry of this cache) device-resident, stream-ordered on `stream`;
  // does nothing when they already are. Never drops.
  void upload(const DevicePlan& dp, cudaStream_t stream);

  size_t size() const { return plans_.size(); }
  // bumped by every drop: plan pointers taken before it are invalid
  uint64_t generation() const { return generation_; }
  // tables copied to the device so far
  uint64_t uploads() const { return uploads_; }

 private:
  void drop(cudaStream_t stream);
  uint8_t* place(size_t bytes);  // device memory for one plan's tables, from the arena

  size_t max_plans_, max_table_bytes_;
  std::unordered_map<uint64_t, std::unique_ptr<DevicePlan>> plans_;
  size_t table_bytes_ = 0;  // tables of every entry, uploaded or not
  uint64_t generation_ = 1;
  uint64_t uploads_ = 0;
  std::vector<void*> blocks_;           // the arena; tables are placed in the last block
  size_t block_cap_ = 0, block_used_ = 0;
};

}  // namespace cgx

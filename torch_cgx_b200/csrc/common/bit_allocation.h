// Per-layer bit widths under a byte budget: the multiple-choice knapsack behind
// `ops.allocate_bits` and the adaptive native DDP hook. One width per layer, least summed
// quantization error with the summed wire bytes within the budget, by dynamic programming over
// the budget split into `resolution` bins (DESIGN §2.12). Host code, run once per adaptation
// period.
#pragma once
#include <cstdint>
#include <optional>
#include <vector>

namespace cgx {

// Wire bytes of one layer at `bits` with its bucket clamped to [1, kMaxBlockElems] as the plan
// clamps it: 8 bytes of {unit, min} per bucket plus `bits` bytes per pack group of 8 values, every
// bucket starting a fresh group (wire.h: block_num_buckets / block_num_groups). The 16-byte
// alignment of a block record's two sections is left out. bits >= 32: numel * 4.
int64_t layer_wire_bytes(int64_t numel, int bits, int64_t bucket_size);

// errors: row-major [L, K], entry [l, k] the error of layer l at candidates[k].
//  * Costs are layer_wire_bytes, each rounded up to whole bins of (room / resolution) bytes.
//  * target_bits: the uniform width the budget came from; by default the widest candidate whose
//    uniform assignment fits (the narrowest when none fits). If the search ends with more error
//    than the uniform assignment at that width, the uniform assignment comes back.
//  * A layer with a non-finite error keeps current[l] (target_bits without `current`), and its
//    bytes at that width come off the budget.
//  * Ties: the fewest bins that reach the least error; within a layer, candidates are tried in
//    (bytes, index) order and only a strictly smaller error replaces a choice. Equal inputs give
//    equal outputs.
// Returns one width per layer (current.size() entries when `current` is longer than L).
// Throws std::out_of_range when `current` is shorter than L.
std::vector<int> allocate_bits(const double* errors, int64_t L, const std::vector<int64_t>& numels,
                               const std::vector<int64_t>& bucket_sizes, const std::vector<int>& candidates,
                               int64_t budget_bytes, const std::vector<int>* current, int64_t resolution,
                               std::optional<int> target_bits);

}  // namespace cgx

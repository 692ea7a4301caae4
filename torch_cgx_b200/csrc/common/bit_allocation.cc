#include "bit_allocation.h"

#include <algorithm>
#include <cmath>
#include <limits>
#include <numeric>
#include <stdexcept>

#include "wire.h"

namespace cgx {

namespace {

// NumPy's float64 sum of a strided column (pairwise_sum in loops_utils.h): 8 accumulators over
// blocks of at most 128 elements, halves split at multiples of 8. The uniform-width fallback
// compares against this sum, so it has to round exactly as NumPy does.
double pairwise_sum(const double* a, int64_t n, int64_t stride) {
  if (n < 8) {
    double res = 0.;
    for (int64_t i = 0; i < n; ++i) res += a[i * stride];
    return res;
  }
  if (n <= 128) {
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = a[j * stride];
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
      for (int j = 0; j < 8; ++j) r[j] += a[(i + j) * stride];
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i * stride];
    return res;
  }
  int64_t n2 = n / 2;
  n2 -= n2 % 8;
  return pairwise_sum(a, n2, stride) + pairwise_sum(a + n2 * stride, n - n2, stride);
}

}  // namespace

int64_t layer_wire_bytes(int64_t numel, int bits, int64_t bucket_size) {
  if (bits >= kRawBits) return numel * 4;
  const int64_t b = std::max<int64_t>(1, std::min<int64_t>(bucket_size, kMaxBlockElems));
  const int64_t nb = (numel + b - 1) / b;
  const int64_t groups = numel / b * ((b + 7) / 8) + (numel % b + 7) / 8;
  return nb * 8 + groups * bits;
}

std::vector<int> allocate_bits(const double* errors, int64_t L, const std::vector<int64_t>& numels,
                               const std::vector<int64_t>& bucket_sizes, const std::vector<int>& candidates,
                               int64_t budget_bytes, const std::vector<int>* current, int64_t resolution,
                               std::optional<int> target_bits) {
  const int64_t K = (int64_t)candidates.size();
  std::vector<int64_t> cost((size_t)(L * K));
  for (int64_t l = 0; l < L; ++l)
    for (int64_t k = 0; k < K; ++k) cost[l * K + k] = layer_wire_bytes(numels[l], candidates[k], bucket_sizes[l]);
  auto column_cost = [&](int64_t k) {
    int64_t s = 0;
    for (int64_t l = 0; l < L; ++l) s += cost[l * K + k];
    return s;
  };
  if (!target_bits) {
    std::optional<int> widest;
    for (int64_t k = 0; k < K; ++k)
      if (column_cost(k) <= budget_bytes && (!widest || candidates[k] > *widest)) widest = candidates[k];
    target_bits = widest ? *widest : *std::min_element(candidates.begin(), candidates.end());
  }
  const int target = *target_bits;
  if (current && (int64_t)current->size() < L)
    throw std::out_of_range("allocate_bits: current has fewer entries than there are layers");
  const std::vector<int> keep = current ? *current : std::vector<int>((size_t)L, target);

  std::vector<int64_t> free;  // layers whose error row is finite
  int64_t fixed_bytes = 0;
  for (int64_t l = 0; l < L; ++l) {
    bool finite = true;
    for (int64_t k = 0; k < K; ++k) finite = finite && std::isfinite(errors[l * K + k]);
    if (finite)
      free.push_back(l);
    else
      fixed_bytes += layer_wire_bytes(numels[l], keep[l], bucket_sizes[l]);
  }
  const int64_t room = budget_bytes - fixed_bytes;
  const auto kt_it = std::find(candidates.begin(), candidates.end(), target);
  const int64_t k_t = kt_it == candidates.end() ? -1 : (int64_t)(kt_it - candidates.begin());
  std::vector<int> uniform = keep;
  for (int64_t l : free) uniform[l] = target;
  const int64_t F = (int64_t)free.size();
  if (F == 0 || room <= 0) return uniform;

  // bins[i, k] = ceil(cost * R / room): any choice with sum(bins) <= R fits the room
  const int64_t R = resolution;
  std::vector<int64_t> bins((size_t)(F * K));
  std::vector<double> e((size_t)(F * K));  // the error rows of the free layers, row-major
  for (int64_t i = 0; i < F; ++i)
    for (int64_t k = 0; k < K; ++k) {
      bins[i * K + k] = (cost[free[i] * K + k] * R + room - 1) / room;
      e[i * K + k] = errors[free[i] * K + k];
    }
  std::vector<int64_t> order((size_t)K);
  std::vector<double> dp((size_t)R + 1, 0.0), best((size_t)R + 1);  // least error within c bins
  std::vector<int16_t> choice((size_t)(F * (R + 1)));
  const double inf = std::numeric_limits<double>::infinity();
  for (int64_t i = 0; i < F; ++i) {
    // candidates in (bytes, index) order with strict improvement: ties keep fewer bytes
    const int64_t* ci = &cost[free[i] * K];
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return ci[a] < ci[b]; });
    std::fill(best.begin(), best.end(), inf);
    int16_t* pick = &choice[(size_t)(i * (R + 1))];
    for (int64_t k : order) {
      const int64_t c = bins[i * K + k];
      if (c > R) continue;
      const double ek = e[i * K + k];
      for (int64_t j = c; j <= R; ++j) {
        const double v = dp[j - c] + ek;
        if (v < best[j]) {
          best[j] = v;
          pick[j] = (int16_t)k;
        }
      }
    }
    dp.swap(best);
  }
  if (!std::isfinite(dp[R])) return uniform;
  int64_t c = 0;  // fewest bins that reach the least error
  while (!(dp[c] == dp[R])) ++c;
  const double total = dp[R];
  std::vector<int> out = keep;
  for (int64_t i = F - 1; i >= 0; --i) {
    const int64_t k = choice[(size_t)(i * (R + 1) + c)];
    out[free[i]] = candidates[k];
    c -= bins[i * K + k];
  }
  if (k_t >= 0) {
    int64_t uniform_cost = 0;
    for (int64_t l : free) uniform_cost += cost[l * K + k_t];
    if (uniform_cost <= room && total > pairwise_sum(&e[k_t], F, K)) return uniform;
  }
  return out;
}

}  // namespace cgx

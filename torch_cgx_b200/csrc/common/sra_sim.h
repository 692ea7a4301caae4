// Single-process, W-rank simulation of the compressed Scatter-Reduce-AllGather
// on CPU memory. Performs exactly the arithmetic of the fused CUDA kernel
// (same plan, same block primitives, same summation order, same RNG streams),
// so tests can demand bit-equality between the GPU result and this oracle.
// Numerics spec: SURVEY.md §2.7 ("SRA numerics"),
// /root/reference/src/common/scatter_reduce_allgather.cc:143-160.
#pragma once
#include <cstdint>
#include <vector>
#include "philox.h"
#include "plan.h"
#include "quant_math.h"

namespace cgx {

struct RngParams {
  uint64_t seed = 0;
  uint32_t seq = 0;
  bool stochastic = false;
};

inline RngKey make_rng_key(const RngParams& r, int rank, int phase) {
  RngKey k;
  k.seed_lo = (uint32_t)r.seed;
  k.seed_hi = (uint32_t)(r.seed >> 32);
  k.seq = r.seq;
  k.stream = (uint32_t)rank * 2u + (uint32_t)phase;
  k.enabled = r.stochastic ? 1u : 0u;
  return k;
}

// bufs[r] = base pointer of rank r's tensor (dtype plan.dtype), reduced in place.
// An FP8 `codec` (8-bit plans; raw blocks are the same either way): chunk c's owner sums
// fl(x_c * prescale) and, for every q != c in rank order, fl(float(code_q) * unit_q) of the FP8
// record of fl(x_q * prescale), each add rounded on its own; the fp32 sum is encoded once and every
// rank stores the values decoded from those codes. The SR codecs draw phase A's bits from stream
// q * 2 and phase B's from c * 2 + 1, as max-min's stochastic rounding does.
void sra_simulate(const Plan& plan, const std::vector<void*>& bufs, float prescale, const RngParams& rng,
                  WireCodec codec = kMaxMin);

// One-shot allreduce oracle: result = T( sum over ranks r (in order) of decode(Q_r(x_r * prescale)) ),
// every contribution quantized exactly once; `plan` must be a single-chunk plan (world == 1).
// An FP8 `codec`: Q_r is the FP8 record (an SR codec: stream r * 2) and the sum starts from +0.
void oneshot_simulate(const Plan& plan, const std::vector<void*>& bufs, float prescale, const RngParams& rng,
                      WireCodec codec = kMaxMin);

// Reduce-scatter oracle (rs_kernel): `plan` covers a shard table replicated W times at stride
// `shard` elements, so chunk c is copy c. out_bufs[c][e - c * shard] = T(prescale * in_c[e] + sum over
// q != c, in rank order, of decode(Q_q(prescale * in_q[e]))) for every element e of chunk c: the
// allreduce's phase-B sum (same primitives, order and phase-A RNG streams), not requantized.
void reduce_scatter_simulate(const Plan& plan, const std::vector<const void*>& in_bufs,
                             const std::vector<void*>& out_bufs, uint64_t shard, float prescale,
                             const RngParams& rng, WireCodec codec = kMaxMin);

// All-to-all oracle (a2a_kernel): counts[q][r] elements go from rank q to rank r. Rank q's chunks
// lie in in_bufs[q] in destination order, rank r's output holds the chunks in source order. The own
// chunk is copied, and so is every chunk when bits >= kRawBits (raw). Every other chunk is decode(Q(x))
// with buckets counted from the chunk's first element (common/a2a.h) and the pair's random stream
// a2a_rng_stream(q, r). With an FP8 codec (bits 8) the chunks use its records instead of max-min's
// (an SR codec: the pair's stream, the own chunk's a2a_rng_stream(r, r) with codes). With `out_scales` (one per rank; an FP8 codec, bucket <= kMaxBlockElems
// dividing every count) out_bufs[r] receives one code byte per element and out_scales[r] the unit of
// every bucket, undecoded, the own chunk encoded too (the fused kernel's codes output).
void all_to_all_simulate(int dtype, const std::vector<const void*>& in_bufs, const std::vector<void*>& out_bufs,
                         const std::vector<std::vector<uint64_t>>& counts, int bits, WireCodec codec,
                         uint32_t bucket, const RngParams& rng, const std::vector<float*>* out_scales = nullptr);

// Quantize->dequantize round trip of one rank's buffer through the plan's
// blocks (what a single compression step does to the data); used by the Python
// ops and the tests.
// An FP8 `codec` (8-bit plans) quantizes the compressed blocks with its records (an SR codec with the
// stream rank * 2 + phase); raw blocks are the same either way.
void roundtrip_simulate(const Plan& plan, void* buf, float prescale, const RngParams& rng, int rank, int phase,
                        WireCodec codec = kMaxMin);

// The FP8 records of `plan`'s blocks (every one compressed at 8 bits, buckets dividing the block
// offsets) of the values in `src`, left undecoded: codes[elem_off + i] = element i's code and
// scales[elem_off / bucket + b] the unit of its bucket b (the all-gather's codes output); an SR codec
// draws its bits from `rng`.
void codes_simulate(const Plan& plan, const void* src, uint8_t* codes, float* scales, WireCodec codec,
                    const RngKey& rng);

}  // namespace cgx

#include "sra_sim.h"

#include <cstring>
#include <stdexcept>

#include "a2a.h"

#include "block_ops.h"

namespace cgx {

void sra_simulate(const Plan& plan, const std::vector<void*>& bufs, float prescale, const RngParams& rng,
                  WireCodec codec) {
  const int W = plan.world;
  if ((int)bufs.size() != W) throw std::invalid_argument("sra_simulate: need one buffer per rank");
  std::vector<float> acc(kMaxBlockElems), tmp(kMaxBlockElems);
  std::vector<uint8_t> rec(kMaxBlockElems * 4 + 64 + kMaxBlockBuckets * 8 + 64);
  for (int c = 0; c < W; ++c) {
    for (uint32_t b = plan.chunk_begin(c); b < plan.chunk_end(c); ++b) {
      const BlockDesc& d = plan.blocks[b];
      cpu::load_block(bufs[c], plan.dtype, d, prescale, acc.data());
      if (codec != kMaxMin && block_bits(d) < kRawBits) {
        for (int q = 0; q < W; ++q) {
          if (q == c) continue;
          cpu::load_block(bufs[q], plan.dtype, d, prescale, tmp.data());
          cpu::quantize_block_fp8(tmp.data(), d, rec.data(), codec, make_rng_key(rng, q, 0));
          cpu::decode_block_fp8_add(rec.data(), d, acc.data(), codec);
        }
        cpu::quantize_block_fp8(acc.data(), d, rec.data(), codec, make_rng_key(rng, c, 1));
        for (int p = 0; p < W; ++p) cpu::decode_block_fp8_store(rec.data(), plan.dtype, d, bufs[p], codec);
        continue;
      }
      for (int q = 0; q < W; ++q) {
        if (q == c) continue;
        cpu::load_block(bufs[q], plan.dtype, d, prescale, tmp.data());
        cpu::quantize_block(tmp.data(), plan.dtype, d, rec.data(), make_rng_key(rng, q, 0), b);
        cpu::decode_block_add(rec.data(), plan.dtype, d, acc.data());
      }
      cpu::quantize_block(acc.data(), plan.dtype, d, rec.data(), make_rng_key(rng, c, 1), b);
      for (int p = 0; p < W; ++p) cpu::decode_block_store(rec.data(), plan.dtype, d, bufs[p]);
    }
  }
}

void reduce_scatter_simulate(const Plan& plan, const std::vector<const void*>& in_bufs,
                             const std::vector<void*>& out_bufs, uint64_t shard, float prescale,
                             const RngParams& rng, WireCodec codec) {
  const int W = plan.world;
  if ((int)in_bufs.size() != W || (int)out_bufs.size() != W)
    throw std::invalid_argument("reduce_scatter_simulate: need one input and one output per rank");
  std::vector<float> acc(kMaxBlockElems), tmp(kMaxBlockElems);
  std::vector<uint8_t> rec(kMaxBlockElems * 4 + 64 + kMaxBlockBuckets * 8 + 64);
  for (int c = 0; c < W; ++c) {
    for (uint32_t b = plan.chunk_begin(c); b < plan.chunk_end(c); ++b) {
      const BlockDesc& d = plan.blocks[b];
      cpu::load_block(in_bufs[c], plan.dtype, d, prescale, acc.data());
      for (int q = 0; q < W; ++q) {
        if (q == c) continue;
        cpu::load_block(in_bufs[q], plan.dtype, d, prescale, tmp.data());
        if (codec != kMaxMin && block_bits(d) < kRawBits) {
          cpu::quantize_block_fp8(tmp.data(), d, rec.data(), codec, make_rng_key(rng, q, 0));
          cpu::decode_block_fp8_add(rec.data(), d, acc.data(), codec);
          continue;
        }
        cpu::quantize_block(tmp.data(), plan.dtype, d, rec.data(), make_rng_key(rng, q, 0), b);
        cpu::decode_block_add(rec.data(), plan.dtype, d, acc.data());
      }
      const uint64_t o = (uint64_t)d.elem_off - (uint64_t)c * shard;
      for (uint32_t i = 0; i < block_n(d); ++i) cpu::store_elem(out_bufs[c], plan.dtype, o + i, acc[i]);
    }
  }
}

void oneshot_simulate(const Plan& plan, const std::vector<void*>& bufs, float prescale, const RngParams& rng,
                      WireCodec codec) {
  if (plan.world != 1) throw std::invalid_argument("oneshot_simulate: plan must have a single chunk");
  const int W = (int)bufs.size();
  std::vector<float> acc(kMaxBlockElems), tmp(kMaxBlockElems);
  std::vector<uint8_t> rec(kMaxBlockElems * 4 + 64 + kMaxBlockBuckets * 8 + 64);
  for (uint32_t b = 0; b < plan.blocks.size(); ++b) {
    const BlockDesc& d = plan.blocks[b];
    const uint32_t n = block_n(d);
    for (uint32_t i = 0; i < n; ++i) acc[i] = 0.f;
    for (int q = 0; q < W; ++q) {
      cpu::load_block(bufs[q], plan.dtype, d, prescale, tmp.data());
      if (codec != kMaxMin && block_bits(d) < kRawBits) {
        cpu::quantize_block_fp8(tmp.data(), d, rec.data(), codec, make_rng_key(rng, q, 0));
        cpu::decode_block_fp8_add(rec.data(), d, acc.data(), codec);
        continue;
      }
      cpu::quantize_block(tmp.data(), plan.dtype, d, rec.data(), make_rng_key(rng, q, 0), b);
      cpu::decode_block_add(rec.data(), plan.dtype, d, acc.data());
    }
    for (int p = 0; p < W; ++p)
      for (uint32_t i = 0; i < n; ++i) cpu::store_elem(bufs[p], plan.dtype, (uint64_t)d.elem_off + i, acc[i]);
  }
}

void all_to_all_simulate(int dtype, const std::vector<const void*>& in_bufs, const std::vector<void*>& out_bufs,
                         const std::vector<std::vector<uint64_t>>& counts, int bits, WireCodec codec,
                         uint32_t bucket, const RngParams& rng, const std::vector<float*>* out_scales) {
  const int W = (int)in_bufs.size();
  if ((int)out_bufs.size() != W || (int)counts.size() != W)
    throw std::invalid_argument("all_to_all_simulate: need one input, output and count row per rank");
  for (const auto& row : counts)
    if ((int)row.size() != W) throw std::invalid_argument("all_to_all_simulate: counts must be W x W");
  const bool codes = out_scales != nullptr;
  if (codes) {
    if ((int)out_scales->size() != W) throw std::invalid_argument("all_to_all_simulate: need one scales buffer per rank");
    if (codec == kMaxMin || bits != 8) throw std::invalid_argument("all_to_all_simulate: codes need an FP8 codec");
    if (bucket < 1 || bucket > kMaxBlockElems) throw std::invalid_argument("all_to_all_simulate: bad bucket for codes");
    for (const auto& row : counts)
      for (uint64_t n : row)
        if (n % bucket) throw std::invalid_argument("all_to_all_simulate: with codes every count holds whole buckets");
  }
  const int es = dtype_size(dtype);
  std::vector<float> acc(kMaxBlockElems);
  std::vector<uint8_t> rec(kMaxBlockElems * 4 + 64 + kMaxBlockBuckets * 8 + 64);
  for (int q = 0; q < W; ++q) {
    uint64_t in_off = 0;
    for (int r = 0; r < W; ++r) {
      uint64_t out_off = 0;
      for (int s = 0; s < q; ++s) out_off += counts[s][r];
      const uint64_t n = counts[q][r];
      const uint8_t* src = static_cast<const uint8_t*>(in_bufs[q]) + in_off * es;
      uint8_t* dst = static_cast<uint8_t*>(out_bufs[r]) + out_off * (codes ? 1 : es);
      in_off += n;
      if (n == 0) continue;
      if (!codes && (q == r || bits >= kRawBits)) {
        std::memcpy(dst, src, n * es);
        continue;
      }
      if (n >= (1ull << 32)) throw std::invalid_argument("all_to_all_simulate: chunk exceeds 2^32 elements");
      const A2aGeom g = a2a_geom((uint32_t)n, bits, bucket, es);
      RngKey key = make_rng_key(rng, q, 0);
      key.stream = a2a_rng_stream(q, r);
      for (uint32_t b = 0; b < a2a_num_blocks(g); ++b) {
        BlockDesc d;
        d.elem_off = b * g.block_elems;
        d.wire_off = 0;
        d.n_bits = (a2a_block_n(g, b) & 0xFFFFFFu) | ((uint32_t)g.bits << 24);
        d.bucket = g.bucket;
        cpu::load_block(src, dtype, d, 1.0f, acc.data());
        if (codes) {
          cpu::quantize_block_fp8(acc.data(), d, rec.data(), codec, key);
          cpu::unpack_block_fp8(rec.data(), d, dst, (*out_scales)[r] + out_off / bucket);
          continue;
        }
        if (codec != kMaxMin) {
          cpu::quantize_block_fp8(acc.data(), d, rec.data(), codec, key);
          cpu::decode_block_fp8_store(rec.data(), dtype, d, dst, codec);
          continue;
        }
        cpu::quantize_block(acc.data(), dtype, d, rec.data(), key, b);
        cpu::decode_block_store(rec.data(), dtype, d, dst);
      }
    }
  }
}

void roundtrip_simulate(const Plan& plan, void* buf, float prescale, const RngParams& rng, int rank, int phase,
                        WireCodec codec) {
  std::vector<float> acc(kMaxBlockElems);
  std::vector<uint8_t> rec(kMaxBlockElems * 4 + 64 + kMaxBlockBuckets * 8 + 64);
  for (uint32_t b = 0; b < plan.blocks.size(); ++b) {
    const BlockDesc& d = plan.blocks[b];
    cpu::load_block(buf, plan.dtype, d, prescale, acc.data());
    if (codec != kMaxMin && block_bits(d) < kRawBits) {
      cpu::quantize_block_fp8(acc.data(), d, rec.data(), codec, make_rng_key(rng, rank, phase));
      cpu::decode_block_fp8_store(rec.data(), plan.dtype, d, buf, codec);
      continue;
    }
    cpu::quantize_block(acc.data(), plan.dtype, d, rec.data(), make_rng_key(rng, rank, phase), b);
    cpu::decode_block_store(rec.data(), plan.dtype, d, buf);
  }
}

void codes_simulate(const Plan& plan, const void* src, uint8_t* codes, float* scales, WireCodec codec,
                    const RngKey& rng) {
  if (codec == kMaxMin) throw std::invalid_argument("codes_simulate: needs an FP8 codec");
  std::vector<float> acc(kMaxBlockElems);
  std::vector<uint8_t> rec(kMaxBlockElems * 4 + 64 + kMaxBlockBuckets * 8 + 64);
  for (const BlockDesc& d : plan.blocks) {
    if (block_bits(d) != 8 || d.elem_off % d.bucket)
      throw std::invalid_argument("codes_simulate: needs 8-bit blocks that start on a bucket boundary");
    cpu::load_block(src, plan.dtype, d, 1.0f, acc.data());
    cpu::quantize_block_fp8(acc.data(), d, rec.data(), codec, rng);
    cpu::unpack_block_fp8(rec.data(), d, codes, scales);
  }
}

}  // namespace cgx

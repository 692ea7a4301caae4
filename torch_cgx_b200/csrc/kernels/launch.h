// Host-callable launchers of every CUDA kernel in the framework (no torch
// dependency: these TUs compile in seconds and are what `cuobjdump -sass`
// inspects).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "../common/a2a.h"
#include "../common/philox.h"
#include "../common/wire.h"

namespace cgx {

// Device-resident call counter of one heap: the epoch of a launch is read from here by every
// CTA and bumped by the last CTA to finish, so a captured CUDA graph replays with fresh epochs
// (kernel arguments are frozen at capture time).
struct DeviceSync {
  uint32_t epoch;     // number of completed fused launches on this heap
  uint32_t finished;  // CTAs of the running launch that are done
  uint32_t pad[2];
};

// ---- fused Scatter-Reduce-AllGather / one-shot over peer memory ------------
struct SraParams {
  void* data;                    // this rank's gradient buffer (T*), reduced in place
  const WarpItem* items;         // device plan: flattened warp items ...
  const uint32_t* item_first;    // ... and the first item of every (chunk, lane) slot [world*lanes + 1]
  int rank;
  int world;
  int lanes;                     // == gridDim.x
  int dtype;
  uint32_t epoch_hint;           // host mirror of the epoch this launch will get (== device epoch
                                 // outside graph replay; only used to advance the RNG sequence)
  float prescale;                // gradients are multiplied by this before anything else (1/W for AVG)
  RngKey rng;                    // .stream is filled in by the kernel
  uint32_t slot_bytes;           // stride between per-source slots inside recv1/recv2
  uint32_t flag_stride;          // lanes capacity of the flag arrays
  uint32_t os_parity_stride;     // one-shot: byte distance between the two alternating regions
  uint8_t* recv1[kMaxPeers];     // recv1[p]: base of rank p's phase-1 receive region (peer-mapped)
  uint8_t* recv2[kMaxPeers];     // recv2[p]: base of rank p's phase-2 receive region
  uint32_t* flags1[kMaxPeers];   // flags1[p][src*flag_stride + lane]
  uint32_t* flags2[kMaxPeers];
  uint8_t* mc_recv1;             // NVLS multicast aliases of the same regions (nullptr: unicast only)
  uint8_t* mc_recv2;
  int mc_reduce;                 // raw items are reduced inside the switch (multimem.ld_reduce)
  uint32_t* status;              // local error word (0 = ok), host-mapped
  const uint32_t* abort_word;    // host-mapped: non-zero = stop waiting for peers (ProcessGroup::abort)
  uint64_t timeout_ns;
  DeviceSync* sync;
  unsigned long long* trace;     // optional [lanes][8] device timestamps (ns, globaltimer), nullptr = off
  int uniform_bits;              // common bits of all compressed items (2/4/8 select a specialised kernel), else 0
  int slice_elems;               // 512 or 1024 (plan.slice_elems)
  int oneshot;                   // 0: three-phase SRA, 1: one-shot
  int stages;                    // SRA: pieces every chunk is pipelined in (1..4, stages * world <= 32)
  void* out;                     // reduce-scatter: output shard (T*); all-gather: gathered output (T*);
                                 // nullptr for the allreduce kernels
  uint64_t out_shift;            // reduce-scatter: element of `data` that lands on out[0];
                                 // all-gather: element of `out` that data[0] lands on (rank * shard stride)
  int gather;                    // with `out`: 1 = all-gather, 0 = reduce-scatter
  int codec;                     // WireCodec of the compressed items (common/quant_math.h); an FP8 codec
                                 // needs uniform_bits 8
  // all-gather only. nullptr: `out` receives the decoded values (T). Otherwise (an FP8 codec, every
  // item compressed) `out` receives one FP8 code byte per element and out_scales[e / out_bucket] the
  // unit of the bucket starting at output element e, for every chunk; the own chunk holds the bytes
  // its owner published.
  float* out_scales;
  uint32_t out_bucket;
};

constexpr int kSraThreads = 256;
constexpr int kSraWarps = kSraThreads / 32;
constexpr int kSraCtasPerSm = 2;
// kSraBadIndex: the routed all-to-all met an index naming a row outside its tensor, or (the combine)
// an output_index naming one slot twice; the status word then holds (rank << 8) | which << 16
// instead of the peer and the lane, which = 0 input_index, 1 output_index, 2 a repeated slot
enum SraStatus : uint32_t { kSraOk = 0, kSraTimeoutPhase1 = 1, kSraTimeoutPhase2 = 2, kSraAborted = 3, kSraBadIndex = 4 };

// max CTAs of the fused kernel that can be co-resident on the current device
int sra_max_resident_ctas(int dtype);
// p.out != nullptr: all-gather (p.gather) or reduce-scatter kernel, else p.oneshot selects one-shot /
// three-phase SRA
cudaError_t launch_sra_fused(const SraParams& p, cudaStream_t stream);

// ---- compressed all-to-all (a2a_kernel.cuh) ------------------------------------
// One launch per call, whatever the splits: every chunk's items and windows are derived on the
// device from (elements, bits, bucket, dtype) (common/a2a.h), so nothing is uploaded per call.
struct A2aParams {
  const void* in;                  // T*: my chunks, in destination order
  void* out;                       // T*: the chunks I receive, in source order
  uint32_t in_off[kMaxPeers];      // my chunk for rank q: elements [in_off[q], in_off[q] + in_cnt[q]) of `in`
  uint32_t in_cnt[kMaxPeers];
  uint32_t out_off[kMaxPeers];     // rank q's chunk for me: elements [out_off[q], + out_cnt[q]) of `out`
  uint32_t out_cnt[kMaxPeers];
  int rank;
  int world;
  int lanes;                       // == gridDim.x, the same on every rank
  int dtype;
  int bits;                        // 1..8, or >= 32 for raw
  uint32_t bucket;                 // as requested (a2a_geom clamps it)
  uint32_t epoch_hint;             // host mirror of the epoch (advances the RNG sequence on graph replay)
  RngKey rng;                      // .stream is filled in per pair (a2a_rng_stream)
  uint32_t slot_bytes;             // stride between per-source slots inside recv
  uint32_t lane_slot;              // a lane's share of a slot (a2a_lane_slot_bytes)
  uint32_t flag_stride;
  uint8_t* recv[kMaxPeers];        // recv[p]: base of rank p's recv1 region (peer-mapped)
  uint32_t* flags2[kMaxPeers];     // closing handshake, as rs_kernel / ag_kernel
  uint64_t* landed[kMaxPeers];     // landed[p][src * flag_stride + lane]: window of src landed in p's slot
  uint64_t* released[kMaxPeers];   // released[p][dst * flag_stride + lane]: dst is done with p's window
  uint32_t* status;
  const uint32_t* abort_word;
  uint64_t timeout_ns;
  DeviceSync* sync;
  // Routed form (launched only when a2a_rows_fit(row, bits, bucket, dtype)): the offsets and counts
  // above are those of the logical buffers of whole rows of `row` elements; row i of the logical
  // send buffer is row in_index[i] of `in` (in_rows rows), row j of the logical receive buffer is
  // row out_index[j] of `out` (out_rows rows). A nullptr index: that side is the logical buffer.
  const int64_t* in_index;
  const int64_t* out_index;
  uint32_t row;
  uint64_t in_rows;
  uint64_t out_rows;
  int codec;                       // WireCodec (common/quant_math.h); FP8 codecs need bits 8 (SR codecs: rng)
  // nullptr: `out` receives the decoded values (T). Otherwise (FP8 codecs only) `out` receives one
  // FP8 code byte per element and out_scales[e / bucket] the unit of the bucket starting at output
  // element e, every chunk -- the own one included -- encoded; counts and rows hold whole buckets.
  float* out_scales;
  // Weighted top-k combine (routed, decoded output only; nullptr: none). `out` holds the slots:
  // row s = t * topk + c is choice c of token t. Once every slot row of token t has landed in the
  // columns [seg * span, (seg + 1) * span), the last warp to arrive writes those columns of
  // combine_out[t] = T(fma chain of gate[t, c] * slot row c, c = 0 .. topk - 1) (combine_segment).
  // masks[t * (row / span) + seg] collects the arrived choices, one bit each; zero before the launch.
  void* combine_out;               // T*: [out_rows / topk, row]
  const float* gate;               // [out_rows / topk, topk]
  uint32_t* masks;
  uint32_t topk;                   // 1..32
  uint32_t span;                   // a2a_row_span(bits, bucket, dtype)
  // Scaled send (with in_index, decoded output, no combine; nullptr: none): row i of the logical send
  // buffer is T(x * in_scale[i]), one fp32 multiply rounded to nearest in T, the own rows included.
  const float* in_scale;
  // world rank of local rank 0: the random streams are keyed by world ranks (a2a_rng_stream), so
  // a node's chunks on several nodes use the streams they would use on one node of W ranks
  int rank_base;
};
// defined once per dtype in a2a_{f32,f16,bf16}.cu; launches the routed kernel when p.in_index or
// p.out_index is set
cudaError_t launch_a2a_f32(const A2aParams& p, cudaStream_t stream);
cudaError_t launch_a2a_f16(const A2aParams& p, cudaStream_t stream);
cudaError_t launch_a2a_bf16(const A2aParams& p, cudaStream_t stream);

// ---- cross-node all-to-all (a2a_remote.cu, DESIGN §2.13f) ---------------------------------------
// The chunks one rank sends to (pack) or receives from (unpack) the ranks of other nodes, in one
// launch each. Chunk i has cnt[i] elements at element elem_off[i] of the tensor (pack: `in`,
// unpack: `out`) and its records at byte wire_off[i] of the buffer (pack: `out`, unpack: `in`),
// a2a_chunk_wire bytes of them; item_first is the prefix sum of a2a_chunk_items over the chunks.
// Compressed bits only (1..8; an FP8 codec with 8): raw chunks travel as their bytes.
struct A2aRemoteParams {
  const void* in;
  void* out;
  float* out_scales;               // unpack, FP8 codecs: codes output as A2aParams::out_scales; else nullptr
  int dtype;
  int bits;
  int codec;
  uint32_t bucket;                 // as requested (a2a_geom clamps it)
  RngKey rng;                      // pack: .stream is filled in per chunk (a2a_rng_stream(rank, peer[i]))
  int rank;                        // world rank of this rank
  int nchunks;                     // <= kA2aMaxWorld
  int peer[kA2aMaxWorld];          // world rank of chunk i's destination (pack) or source (unpack)
  uint32_t cnt[kA2aMaxWorld];
  uint64_t elem_off[kA2aMaxWorld];
  uint64_t wire_off[kA2aMaxWorld];
  uint32_t item_first[kA2aMaxWorld + 1];
};
cudaError_t launch_a2a_pack(const A2aRemoteParams& p, cudaStream_t stream);
cudaError_t launch_a2a_unpack(const A2aRemoteParams& p, cudaStream_t stream);

// ---- standalone item kernels (generic reducers, Python ops, tests, cross-node path) ----
// All operate on items [first, first+count) of a device item table; `wire` is the base of the
// chunk's wire slot (records live at wire + item offsets). `slice_elems` / `uniform_bits` are
// the plan's.
struct ItemKernelArgs {
  const WarpItem* items;
  uint32_t first, count;
  int dtype;
  int slice_elems;
  int uniform_bits;
  int codec = 0;  // WireCodec: an FP8 codec needs an 8-bit plan whose items [first, first+count) are all
                  // compressed, and deterministic rounding
};
// wire = quantize(src[T] * prescale)
cudaError_t launch_quantize_items(const ItemKernelArgs& a, const void* src, uint8_t* wire, float prescale,
                                  const RngKey& rng, cudaStream_t stream);
// src is an fp32 scratch laid out like the tensor (index = elem_off - base_elem);
// also writes the self-decoded values into `out` (T, index = elem_off) when out != nullptr.
cudaError_t launch_quantize_items_f32(const ItemKernelArgs& a, const float* src_f32, uint32_t base_elem,
                                      uint8_t* wire, const RngKey& rng, void* out, cudaStream_t stream);
// dst[T] = decode(wire)
cudaError_t launch_dequantize_items(const ItemKernelArgs& a, const uint8_t* wire, void* dst, cudaStream_t stream);
// an FP8 plan's records undecoded (any dtype, a.codec ignored): codes[elem_off + i] = the code of
// element i of an item, scales[elem_off / bucket + b] = the unit of its bucket b
cudaError_t launch_unpack_items_fp8(const ItemKernelArgs& a, const uint8_t* wire, uint8_t* codes, float* scales,
                                    uint32_t bucket, cudaStream_t stream);
// acc_f32[elem_off - base_elem + i] = float(init_src[elem_off + i]) * prescale   (init_src != nullptr)
// acc_f32[...] += decode(wire)                                                   (wire != nullptr)
// (an FP8 codec adds fl(float(code) * unit), a separate rounding)
cudaError_t launch_accumulate_items_f32(const ItemKernelArgs& a, const uint8_t* wire, float* acc_f32,
                                        uint32_t base_elem, const void* init_src, float prescale,
                                        cudaStream_t stream);

// ---- weighted top-k combine of slot rows (combine_rows_kernel, the combine's composed path) ----
// out[t, h] = T(acc) with acc = g_0 * x_0, then acc = fma(g_c, x_c, acc) for c = 1 .. k - 1, where
// x_c = float(slots[t * k + c, h]) and g_c = gate[t, c]; slots [T * k, H], gate [T, k] fp32, out [T, H]
cudaError_t launch_combine_rows(const void* slots, const float* gate, void* out, int dtype, uint64_t T, uint32_t k,
                                uint32_t H, cudaStream_t stream);
// The gradient of that combine with respect to the gate (combine_gate_grad_kernel, DESIGN §2.13e):
// grad_gate[t, c] = sum over h of float(grad_out[t, h]) * float(slots[t * k + c, h]) in fp32, in a
// fixed order: lane l = (h / V) % 32 (V = 16 / sizeof(T)) runs acc = fma(go_h, x_h, acc) from +0
// over its elements in increasing h, then acc += shfl_xor(acc, m) for m = 16, 8, 4, 2, 1.
// grad_out [T, H], slots [T * k, H] and grad_gate [T, k] (fp32) contiguous, k 1..32; grad_out and
// slots at any element alignment.
cudaError_t launch_combine_gate_grad(const void* grad_out, const void* slots, float* grad_gate, int dtype, uint64_t T,
                                     uint32_t k, uint32_t H, cudaStream_t stream);
// rows[i, h] = T(float(rows[i, h]) * scale[i]) in place, rows [R, H] contiguous: the scaled send of
// the routed all-to-all's composed path, with the fused kernel's rounding
cudaError_t launch_scale_rows(void* rows, const float* scale, int dtype, uint64_t R, uint64_t H, cudaStream_t stream);

// ---- elementwise helpers (K4/K7 of the reference) ---------------------------
cudaError_t launch_scale_inplace(void* data, int dtype, uint64_t n, float scale, cudaStream_t stream);
cudaError_t launch_add(const void* x, const void* y, void* sum, int dtype, uint64_t n, cudaStream_t stream);
cudaError_t launch_convert(const void* src, int src_dtype, void* dst, int dst_dtype, uint64_t n,
                           cudaStream_t stream);

// ---- ResNet residual join (residual_relu.cu): n elements of dense storage, all operands alike ----
// y = relu(a + b)
cudaError_t launch_residual_relu_forward(const void* a, const void* b, void* y, int dtype, uint64_t n,
                                         cudaStream_t stream);
// g = (y <= 0) ? 0 : ga + gb, or ga alone when gb == nullptr
cudaError_t launch_residual_relu_backward(const void* y, const void* ga, const void* gb, void* g, int dtype,
                                          uint64_t n, cudaStream_t stream);

// ---- training BatchNorm on channels_last input (batchnorm_cl.cu), bit-identical to ATen's kernels ----
struct BnForwardArgs {
  const void* x;  // [M][C], dtype
  void* y;        // like x
  int dtype, M, C;
  const float *weight, *bias;
  float *running_mean, *running_var;  // updated in place
  float *save_mean, *save_invstd;     // [C]
  double momentum, eps;
  bool relu;        // y = relu_(bn(x)) instead of bn(x)
  float* staging;   // 3 * batchnorm_cl_grid_y(M, C) * C floats when that grid is > 1
  int* sem;         // sem_len zeroed ints, left zeroed; launches that share them must be stream-ordered
  int sem_len;      // >= C / 4 + 1
};
struct BnBackwardArgs {
  const void* g;  // gradient of y, like x
  const void* x;
  void* gx;       // like x
  int dtype, M, C;
  const float *weight, *bias, *mean, *invstd;  // mean, invstd: the forward's save_mean, save_invstd
  float *sum_dy, *sum_dy_xmu, *grad_weight, *grad_bias;  // [C]
  bool relu;        // the forward fused the ReLU: g is masked where the forward's output is +0
  float* staging;   // 2 * batchnorm_cl_grid_y(M, C) * C floats when that grid is > 1
  int* sem;         // as for the forward
  int sem_len;
};
int batchnorm_cl_grid_y(int M, int C);
// statistics + running-stat update + invstd, then the transform (with the fused ReLU)
cudaError_t launch_batchnorm_cl_forward(const BnForwardArgs& args, cudaStream_t stream);
// reduction (sum_dy, sum_dy_xmu, grad_weight, grad_bias), then grad_input
cudaError_t launch_batchnorm_cl_backward(const BnBackwardArgs& args, cudaStream_t stream);

// ---- quantization-error estimate of a layer table (quant_error.cu, common/quant_error.h) ----
struct QErrLayer;
struct QErrArgs {
  const void* data;               // flat gradient, dtype
  int dtype;
  const QErrLayer* layer_table;   // [layers] device
  const uint64_t* first;          // [layers + 1] device: first bucket of every layer (qerr_first)
  uint64_t nbuckets;              // first[layers], also on the host: the buckets of one chunk
  int layers;
  const int* bits;           // [K] host: candidate widths, 1..8
  int K;                     // 1..8
  float prescale;
  bool stochastic;
  float* partial;            // [included chunks * nbuckets * K] device scratch
  double* out;               // [layers * K] device
  // sharded mode (common/quant_error.h): `chunks` copies of the layer table at stride chunk_stride
  // elements, chunk skip_chunk left out (-1: none); row l sums the included chunks
  int chunks = 1;
  uint64_t chunk_stride = 0;
  int skip_chunk = -1;
};
cudaError_t launch_quantization_error(const QErrArgs& args, cudaStream_t stream);

}  // namespace cgx

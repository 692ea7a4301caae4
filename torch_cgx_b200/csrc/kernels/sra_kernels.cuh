// The product: ONE kernel per fusion buffer that performs the whole compressed
// Scatter-Reduce-AllGather allreduce over NVLink 4 / NVSwitch.
//
//   phase A  for every peer p: quantize my copy of chunk p item by item and store the packed
//            words straight into p's receive slot (peer-mapped st.global), then ONE system-scope
//            release per lane
//   phase B  acquire the W-1 incoming copies of MY chunk, dequantize + accumulate them with my
//            raw values in fp32 registers, requantize, publish the packed result to every rank
//            -- ONE multimem.st into the NVLS multicast mapping when the heap has one, W-1 peer
//            stores otherwise -- and write the self-decoded values to my gradient buffer
//   phase C  acquire each peer's reduced chunk (in order of arrival), dequantize into my buffer
//
// rs_kernel (reduce-scatter) is phases A and B without the requantization, the publish and phase C.
// ag_kernel (all-gather) is the publish of phase B (of my unreduced shard) and phase C on recv1.
//
// The grid is G persistent *lanes* (CTAs of 8 warps, two per SM). Lane c of every rank only ever
// talks to lane c of the other ranks through single-writer epoch flags, so there is no grid-wide
// or host synchronisation anywhere and lanes pipeline independently. The work of a lane is a
// flat list of warp items (common/wire.h) dealt round-robin to its warps; the hot loops contain
// only the full-slice path (item_ops.cuh), everything rare is out of line.
//
// The epoch lives in device memory (DeviceSync): the kernel is CUDA-graph capturable.
//
// Uncompressed layers ride the same launch as raw items: the classic two-shot P2P allreduce with
// the 1/W prescale fused, or -- with a multicast heap -- an in-switch reduction
// (multimem.ld_reduce + multimem.st), the NVLS algorithm of NCCL inside our kernel.
//
// Reference behaviour being replaced (4-5 launches per layer + host polling):
//   /root/reference/src/common/scatter_reduce_allgather.cc:94-202 (compressed), :308-413 (raw)
//   /root/reference/src/common/nccl_reduce.cc:103-198
//   /root/reference/src/common/shm_communicator.cc:110-177
#pragma once
#include "item_ops.cuh"
#include "launch.h"

namespace cgx {
namespace dev {

// Tracing: per-lane phase timestamps (slot 0: kernel start [min], 1: phase A stores issued,
// 2: phase B inputs arrived, 3: phase B stores issued, 4: last phase-C wait satisfied, 5: end [max],
// 6 / 7: warp 0 after the release (system fence + flag stores) of phase A / B).
__device__ __forceinline__ void trace_mark(const SraParams& p, int lane, int slot, bool is_min = false) {
  unsigned long long* trace = p.trace;
  if (trace == nullptr || (threadIdx.x & 31u) != 0) return;
  const unsigned long long t = globaltimer_ns();
  if (is_min)
    atomicMin(&trace[(size_t)lane * 8 + slot], t);
  else
    atomicMax(&trace[(size_t)lane * 8 + slot], t);
}

// Every CTA reads the epoch before any CTA can have bumped it: the bump happens after ALL CTAs
// of the launch have passed their read (each counts itself as finished only at its very end).
__device__ __forceinline__ void sync_finish(DeviceSync* sync, uint32_t epoch, int lanes) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&sync->finished, 1u) + 1u == (uint32_t)lanes) {
      sync->finished = 0;
      sync->epoch = epoch;
      __threadfence();
    }
  }
}

// warp 0: publish "this lane finished the phase" to every peer. One fence.acq_rel.sys drains the
// NVLink stores of the whole CTA (made visible to this warp by the preceding bar.sync).
__device__ __forceinline__ void signal_peers(uint32_t* const* flags, int W, int r, uint32_t flag_stride, int lane,
                                             uint32_t epoch /* flag_value() */) {
  const uint32_t wl = lane_id();
  if (wl < (uint32_t)W && (int)wl != r) st_release_sys(flags[wl] + (size_t)r * flag_stride + lane, epoch);
}

// warp 0: wait until every peer's flag for this lane reached the epoch. Returns false on timeout
// or abort (and records who was missing in the host-visible status word).
__device__ __forceinline__ bool wait_peers(const uint32_t* my_flags, const SraParams& p, int lane, uint32_t epoch,
                                           uint32_t code) {
  const uint32_t wl = lane_id();
  int rc = 0;
  if (wl < (uint32_t)p.world && (int)wl != p.rank) {
    rc = wait_flag(my_flags + (size_t)wl * p.flag_stride + lane, epoch, p.timeout_ns, p.abort_word);
    if (rc != 0) *p.status = (rc == 2 ? (uint32_t)kSraAborted : code) | (wl << 8) | ((uint32_t)lane << 16);
  }
  return __all_sync(kAll, rc == 0);
}

// ---- per-lane item cache ----------------------------------------------------------------
// The items of ALL chunks of this lane are copied to shared memory once (TMA bulk copies), in the
// order s = 0 (my own chunk), 1, .., W-1 (chunk (rank + s) % W): an item descriptor then costs one
// LDS instead of a dependent global load in front of every data load. Lists longer than the
// cache (huge messages on few lanes) read the remainder from global memory.
//
// Stages: the item list of every chunk is cut into S consecutive pieces. Stage t of the allreduce
// handles piece t of every chunk and has its own flag value, so the NVLink flight time and the
// release/acquire round trip of stage t are hidden behind the computation of stage t+1 (a lane
// pipelines with its peer lanes instead of idling between the phases). The cache is laid out
// stage-major: segment g = t * W + s holds piece t of chunk slot s.
constexpr uint32_t kSmemItems = 1024;
constexpr int kMaxStages = 4;
constexpr int kMaxSegs = 32;  // S * W <= 32: phase C polls one segment per warp lane

struct LaneItems {
  WarpItem items[kSmemItems];
  uint32_t pre[kMaxSegs + 1];    // pre[g]: flat index of the first item of segment g
  uint32_t gfirst[kMaxSegs];     // its index in the global item table
  unsigned long long mbar;       // completion barrier of the bulk copies below
  unsigned long long poll_t0[kSraWarps];  // phase C: when a warp's current flag wait started (0 = not waiting);
                                          // only touched every 1024 polls, so it lives here, not in a register
};

// Flags only ever grow: stage t of call `epoch` publishes epoch * 4 + t + 1.
__device__ __forceinline__ uint32_t flag_value(uint32_t epoch, int stage) {
  return epoch * (uint32_t)kMaxStages + (uint32_t)stage + 1u;
}

// ---- TMA bulk copy (cp.async.bulk, 1-D): global -> shared, completion on an mbarrier -----------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");  // visible to the async proxy
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t tries = 0; !done; ++tries) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (!done && tries > (1u << 24)) __trap();  // a lost copy must not become a silent hang
  }
}

// One elected thread issues ONE bulk copy per segment (each piece of an item list is contiguous in
// the plan table and 16 B granular -- exactly what cp.async.bulk wants); everybody waits on the
// mbarrier.
__device__ __forceinline__ void lane_items_load(LaneItems& li, const SraParams& p, int nchunks, int stages) {
  const int lane = blockIdx.x, G = p.lanes;
  const int nsegs = nchunks * stages;
  if (threadIdx.x < (uint32_t)nsegs) {
    const int t = (int)threadIdx.x / nchunks, s = (int)threadIdx.x - t * nchunks;
    const int q = nchunks == 1 ? 0 : (p.rank + s) % p.world;
    const uint32_t a = p.item_first[q * G + lane];
    const uint32_t n = p.item_first[q * G + lane + 1] - a;
    const uint32_t lo = n * (uint32_t)t / (uint32_t)stages, hi = n * (uint32_t)(t + 1) / (uint32_t)stages;
    li.gfirst[threadIdx.x] = a + lo;
    li.pre[threadIdx.x + 1] = hi - lo;  // count, turned into a prefix below
  }
  if (threadIdx.x == 0) mbar_init(&li.mbar, 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nchunks = nsegs;  // from here on every segment is its own list
    li.pre[0] = 0;
    for (int s = 0; s < nchunks; ++s) li.pre[s + 1] += li.pre[s];
    const uint32_t cached = min(li.pre[nchunks], kSmemItems);
    mbar_expect_tx(&li.mbar, cached * (uint32_t)sizeof(WarpItem));  // 0 bytes: completes at once
    for (int s = 0; s < nchunks; ++s) {
      const uint32_t b = li.pre[s], e = min(li.pre[s + 1], kSmemItems);
      if (e > b) bulk_g2s(&li.items[b], p.items + li.gfirst[s], (e - b) * (uint32_t)sizeof(WarpItem), &li.mbar);
    }
  }
  __syncthreads();  // the prefix table is complete
  mbar_wait(&li.mbar, 0);
}
// item with flat index i, known to belong to segment s
__device__ __forceinline__ WarpItem lane_item(const LaneItems& li, const SraParams& p, uint32_t i, int s) {
  if (i < kSmemItems) return li.items[i];
  return p.items[li.gfirst[s] + (i - li.pre[s])];
}

// Fetch item `i` of a flat range (cursor `s` = its segment, only ever moves forward) and, if it
// is a hot kind with vector-aligned gradients, issue the loads of its values.
// hot: 0 cold item (loads its own data)  1 full slice  2 full raw item.
// Plain scalars / arrays on purpose: a struct here ends up in local memory.
template <typename T, int GPL>
__device__ __forceinline__ void fetch_values(const LaneItems& li, const SraParams& p, uint32_t i, uint32_t end,
                                             WarpItem& it, int& s, int& hot, float (&x)[GPL][8]) {
  hot = 0;
  if (i >= end) return;
  while (i >= li.pre[s + 1]) ++s;
  it = lane_item(li, p, i, s);
  const T* src = reinterpret_cast<const T*>(p.data) + it.elem_off;
  const uint32_t kind = item_kind(it);
  if (!group_aligned<T>(src)) return;
  if (kind == kItemFull) {
    hot = 1;
    slice_load_vec<T, GPL>(src, x);
  } else if (kind == kItemRaw) {
    hot = 2;
    raw_load_vec<T, GPL>(src, x);
  }
}

#define CGX_COPY_WORDS(dst, src)                           \
  _Pragma("unroll") for (int k_ = 0; k_ < GPL; ++k_) {     \
    (dst).lo[k_] = (src).lo[k_];                           \
    (dst).hi[k_] = (src).hi[k_];                           \
    (dst).pm[k_] = (src).pm[k_];                           \
  }

// Each phase is its own out-of-line function: ptxas allocates registers per function, so the
// phase that needs most (B: the words of several sources in flight) does not push the streaming
// phases (A, C: two items at a time) into spilling, and vice versa. Everything a phase needs is
// re-derived from the parameter bank and the shared item cache.
__device__ __forceinline__ RngKey phase_rng(const SraParams& p, uint32_t epoch, uint32_t phase) {
  RngKey rng = p.rng;
  rng.seq += epoch - p.epoch_hint;  // graph replays advance the random stream
  rng.stream = (uint32_t)p.rank * 2u + phase;
  return rng;
}

// ---- phase A: my copy of every other chunk -> its owner. The items of all destinations are dealt
// round-robin to the warps; each warp takes them two at a time (ILP) and pulls the pair after that
// towards L2. With the in-switch reduction the full raw items of ALL chunks (mine included) are
// staged locally. CODEC: the wire codec of the compressed items (the reduce-scatter's FP8 forms).
template <typename T, int KB, int GPL, int CODEC = kMaxMin>
__device__ __forceinline__ void sra_phase_a(const SraParams& p, const LaneItems& li, uint32_t epoch, int stage) {
  const int r = p.rank, W = p.world;
  const int seg0 = stage * W;
  const uint32_t warp = threadIdx.x >> 5;
  T* data = reinterpret_cast<T*>(p.data);
  const RngKey rng = phase_rng(p, epoch, 0u);
  const SrcSet no_src{nullptr, 0u, 0, -1};
  const uint32_t own_end = li.pre[seg0 + 1], total = li.pre[seg0 + W];
  const uint32_t begin = p.mc_reduce ? li.pre[seg0] : own_end;
  auto one = [&](const WarpItem& it, int seg, int hot, float (&x)[GPL][8]) {
    const uint32_t kind = item_kind(it);
    const int cs = seg - seg0;
    const int dstp = (r + cs) % W;
    T* blk = data + it.elem_off;
    if (p.mc_reduce) {
      if (kind == kItemRaw) {
        const OneDst stage{p.recv2[r] + (size_t)dstp * p.slot_bytes};
        if (hot == 2)
          raw_full_x<T, 0, GPL>(x, blk, it, p.prescale, no_src, stage);
        else
          raw_generic<T>(blk, it, p.prescale, no_src, stage, 0);
        return;
      }
      if (cs == 0) return;  // my own chunk: nothing else to send
    }
    const OneDst push{p.recv1[dstp] + (size_t)r * p.slot_bytes};
    if constexpr (CODEC != kMaxMin) {
      if (hot == 1) {
        slice_scale<GPL>(x, p.prescale);
        full_send_fp8_x<CODEC, GPL>(x, it, rng, push);
        return;
      }
      if (kind == kItemFull) {
        full_send_fp8_scaled_unaligned<T, T, CODEC, GPL, false>(blk, it, p.prescale, rng, push, (T*)nullptr);
        return;
      }
      if (kind == kItemBucket) {
        bucket_send_fp8<T, T, CODEC>(blk, it, p.prescale, rng, push, (T*)nullptr);
        return;
      }
    }
    if (hot == 1)
      full_send_x<T, KB, GPL, false, true>(x, it, p.prescale, rng, push, (T*)nullptr);
    else if (hot == 2)
      raw_full_x<T, 0, GPL>(x, blk, it, p.prescale, no_src, push);
    else if (kind == kItemFull)
      full_send_unaligned<T, T, KB, GPL, false>(blk, it, p.prescale, rng, push, (T*)nullptr);
    else if (kind == kItemBucket)
      bucket_quantize<T, T>(blk, it, p.prescale, rng, no_src, push, (T*)nullptr);
    else
      raw_generic<T>(blk, it, p.prescale, no_src, push, 0);
  };
  int sa = seg0 + (p.mc_reduce ? 0 : 1);
  for (uint32_t i = begin + warp; i < total; i += 2 * kSraWarps) {
    WarpItem ita, itb;
    int hota = 0, hotb = 0, sb;
    float xa[GPL][8], xb[GPL][8];
    fetch_values<T, GPL>(li, p, i, total, ita, sa, hota, xa);
    sb = sa;
    const bool has_b = i + kSraWarps < total;
    fetch_values<T, GPL>(li, p, i + kSraWarps, total, itb, sb, hotb, xb);
    {  // next pair -> L2
      int sn = sb;
#pragma unroll
      for (int u = 2; u < 4; ++u) {
        const uint32_t in = i + (uint32_t)u * kSraWarps;
        if (in < total) {
          while (in >= li.pre[sn + 1]) ++sn;
          slice_prefetch_l2<T, GPL>(data + lane_item(li, p, in, sn).elem_off);
        }
      }
    }
    bool done = false;
    if (CODEC == kMaxMin && hota == 1 && hotb == 1 && !(p.mc_reduce && sa == seg0)) {
      const OneDst pa{p.recv1[(r + sa - seg0) % W] + (size_t)r * p.slot_bytes};
      const OneDst pb{p.recv1[(r + sb - seg0) % W] + (size_t)r * p.slot_bytes};
      done = full_send_pair<KB, GPL>(xa, xb, ita, itb, p.prescale, rng, pa, pb);
    }
    if (!done) {
      one(ita, sa, hota, xa);
      if (has_b) one(itb, sb, hotb, xb);
    }
    sa = sb;
  }
}

// ---- phase B: reduce my chunk. The registers of this phase belong to the sources' words (four
// sources in flight); the NEXT item's own values are only pulled towards L2.
// CODEC: the wire codec of the compressed items; an FP8 codec sums the decoded sources, encodes the
// fp32 sum once and keeps the values decoded from its own codes (item_ops.cuh).
template <typename T, int KB, int GPL, int CODEC = kMaxMin>
__device__ __forceinline__ void sra_phase_b(const SraParams& p, const LaneItems& li, uint32_t epoch, int stage) {
  const int r = p.rank, W = p.world;
  const int seg0 = stage * W;
  const uint32_t warp = threadIdx.x >> 5;
  T* data = reinterpret_cast<T*>(p.data);
  const RngKey rng = phase_rng(p, epoch, 1u);
  const uint32_t own_end = li.pre[seg0 + 1];
  const SrcSet ss{p.recv1[r], p.slot_bytes, W, r};
  const MultiDst ds{p.recv2, p.mc_recv2, (uint32_t)r * p.slot_bytes, W, r, nullptr};
  for (uint32_t i = li.pre[seg0] + warp; i < own_end; i += kSraWarps) {
    const WarpItem it = lane_item(li, p, i, seg0);
    const uint32_t kind = item_kind(it);
    T* blk = data + it.elem_off;
    const bool al = group_aligned<T>(blk);
    float x[GPL][8];
    if (al && kind == kItemFull) slice_load_vec<T, GPL>(blk, x);
    if (al && kind == kItemRaw && !p.mc_reduce) raw_load_vec<T, GPL>(blk, x);
    if (i + kSraWarps < own_end) {
      const WarpItem itn = lane_item(li, p, i + kSraWarps, seg0);
      if (!(p.mc_reduce && item_kind(itn) == kItemRaw)) slice_prefetch_l2<T, GPL>(data + itn.elem_off);
    }
    if constexpr (CODEC != kMaxMin) {
      if (kind == kItemFull) {
        if (al)
          full_reduce_fp8_x<T, CODEC, GPL, true>(x, blk, it, p.prescale, rng, ss, ds);
        else
          full_reduce_fp8_unaligned<T, CODEC, GPL>(blk, it, p.prescale, rng, ss, ds);
        continue;
      }
      if (kind == kItemBucket) {
        bucket_reduce_fp8<T, CODEC>(blk, it, p.prescale, rng, ss, ds);
        continue;
      }
    }
    if (kind == kItemFull) {
      if (al)
        full_reduce_x<T, KB, GPL, true>(x, blk, it, p.prescale, rng, ss, ds);
      else
        full_reduce_unaligned<T, KB, GPL>(blk, it, p.prescale, rng, ss, ds);
    } else if (kind == kItemBucket) {
      bucket_quantize<T, T>(blk, it, p.prescale, rng, ss, ds, blk);
    } else if (kind == kItemRaw && p.mc_reduce) {
      raw_full_mc_reduce<T>(blk, it, p.mc_recv2 + (size_t)r * p.slot_bytes);
    } else if (kind == kItemRaw && al) {
      raw_full_x<T, 1, GPL>(x, blk, it, p.prescale, ss, ds);
    } else {
      raw_generic<T>(blk, it, p.prescale, ss, ds, 1);
    }
  }
}

// ---- phase C: decode every peer's reduced chunk, piece by piece in order of arrival. Lane g of
// every warp looks after segment g (polls the flag of its chunk for the value of its stage); the
// items of a segment are dealt to the warps by flat index. Two items per iteration (ILP) with the
// packed words of the NEXT two already in flight.
// AG (the all-gather's decode): the chunks arrive in recv1 under flags1 and are decoded into p.out;
// a timed-out wait also sets *abort_out. AG is a compile-time switch so that the allreduce's
// instantiation is the same code as before it existed. CODEC: the all-gather's wire codec.
// CODES (all-gather, FP8 codec): every item is unpacked into p.out (codes) and p.out_scales instead
// of decoded; the scale index is the item's element in the whole output over p.out_bucket.
template <typename T, int KB, int GPL, bool AG = false, int CODEC = kMaxMin, bool CODES = false>
__device__ __forceinline__ void sra_phase_c(const SraParams& p, const LaneItems& li, uint32_t epoch, int stages,
                                            int* abort_out = nullptr) {
  const int lane = blockIdx.x;
  const int r = p.rank, W = p.world;
  const uint32_t warp = threadIdx.x >> 5, wl = threadIdx.x & 31u;
  T* data = reinterpret_cast<T*>(AG ? p.out : p.data);
  const int my_stage = (int)wl / W, my_slot = (int)wl - my_stage * W;
  const bool mine = my_slot >= 1 && my_stage < stages;
  const uint32_t my_cnt = mine ? li.pre[wl + 1] - li.pre[wl] : 0u;
  const uint32_t* my_flag = (AG ? p.flags1[r] : p.flags2[r]) + (size_t)((r + my_slot) % W) * p.flag_stride + lane;
  uint32_t pending = __ballot_sync(kAll, my_cnt > 0);
  uint32_t spins = 0;
  volatile unsigned long long* t0 = &const_cast<LaneItems&>(li).poll_t0[warp];
  if (wl == 0) *t0 = 0;
  __syncwarp();
  const OneDst none{nullptr};
  while (pending) {
    // the flag value this lane waits for is re-derived on every poll (three compares) instead of
    // occupying a register for the whole phase
    uint32_t w2 = wl;
    asm volatile("" : "+r"(w2));
    const int st = (int)(w2 >= (uint32_t)W) + (int)(w2 >= 2u * (uint32_t)W) + (int)(w2 >= 3u * (uint32_t)W);
    const bool rdy = ((pending >> wl) & 1u) && (int32_t)(ld_acquire_sys(my_flag) - flag_value(epoch, st)) >= 0;
    uint32_t ready = __ballot_sync(kAll, rdy);
    if (!ready) {
      if ((++spins & 0x3FFu) == 0) {
        const uint64_t now = globaltimer_ns();
        if (*t0 == 0) {
          __syncwarp();
          if (wl == 0) *t0 = now;
          __syncwarp();
        }
        const bool aborted = *reinterpret_cast<const volatile uint32_t*>(p.abort_word) != 0;
        if (__any_sync(kAll, aborted || now - *t0 > p.timeout_ns)) {
          if (wl == (uint32_t)__ffs(pending) - 1u)
            *p.status = (aborted ? (uint32_t)kSraAborted : (uint32_t)(AG ? kSraTimeoutPhase1 : kSraTimeoutPhase2)) |
                        ((uint32_t)((r + my_slot) % W) << 8) | ((uint32_t)lane << 16);
          if (AG) *abort_out = 1;
          break;
        }
      }
      continue;
    }
    pending &= ~ready;
    trace_mark(p, lane, 4);
    while (ready) {
      const int s = __ffs(ready) - 1;  // segment
      ready &= ready - 1;
      const int q = (r + __shfl_sync(kAll, my_slot, s)) % W;
      const uint32_t end = li.pre[s + 1];
      const uint8_t* slot = (AG ? p.recv1[r] : p.recv2[r]) + (size_t)q * p.slot_bytes;
      const SrcSet ss{slot, 0u, 1, -1};
      auto fetch = [&](uint32_t i, WarpItem& it, SliceWords<GPL>& w) -> bool {
        if (i >= end) return false;
        it = lane_item(li, p, i, s);
        const bool h = !CODES && item_kind(it) == kItemFull && group_aligned<T>(data + it.elem_off);
        if (h) slice_fetch<KB, GPL>(slot, it.meta_off, it.pay_off, item_lpb_log2(it), KB ? KB : item_bits(it), w);
        return h;
      };
      auto one = [&](const WarpItem& it, const SliceWords<GPL>& w, bool hot) {
        if constexpr (CODES) {
          fp8_unpack_item<GPL>(slot, it, reinterpret_cast<uint8_t*>(p.out) + it.elem_off,
                               p.out_scales + it.elem_off / p.out_bucket);
          return;
        }
        const uint32_t kind = item_kind(it);
        T* blk = data + it.elem_off;
        if constexpr (CODEC != kMaxMin) {
          if (hot) {
            full_recv_fp8_w<T, CODEC, GPL, true>(w, blk);
            return;
          }
          if (kind == kItemFull) {
            full_recv_fp8_unaligned<T, CODEC, GPL>(slot, it, blk);
            return;
          }
          if (kind == kItemBucket) {
            bucket_recv_fp8<T, CODEC>(slot, it, blk);
            return;
          }
        }
        if (hot) {
          full_recv_w<T, KB, GPL, true>(w, it, blk);
        } else if (kind == kItemFull) {
          full_recv_unaligned<T, KB, GPL>(ss, it, blk);
        } else if (AG && (kind == kItemRaw || kind == kItemRawTail)) {
          raw_ag_recv<T>(ss, it, blk);  // the owner's T bits: a -0 must not become 0 + -0 = +0
        } else if (kind == kItemRaw && group_aligned<T>(blk)) {
          float x[2][8];
          raw_full_x<T, 2, 2>(x, blk, it, 1.0f, ss, none);
        } else if (kind == kItemBucket) {
          bucket_recv<T>(ss, it, blk);
        } else {
          raw_generic<T>(blk, it, 1.0f, ss, none, 2);
        }
      };
      uint32_t i = li.pre[s] + ((warp - li.pre[s]) & (kSraWarps - 1));
      WarpItem ita, itb, na, nb;
      SliceWords<GPL> wa, wb, wna, wnb;
      bool hota = fetch(i, ita, wa), hotb = fetch(i + kSraWarps, itb, wb);
      while (i < end) {
        const uint32_t in = i + 2 * kSraWarps;
        const bool hna = fetch(in, na, wna), hnb = fetch(in + kSraWarps, nb, wnb);
        if (CODEC != kMaxMin && hota && hotb) {
          full_recv_fp8_w<T, CODEC, GPL, true>(wa, data + ita.elem_off);
          full_recv_fp8_w<T, CODEC, GPL, true>(wb, data + itb.elem_off);
        } else if (hota && hotb) {
          full_recv_pair<T, KB, GPL>(wa, wb, ita, itb, data + ita.elem_off, data + itb.elem_off);
        } else {
          one(ita, wa, hota);
          if (i + kSraWarps < end) one(itb, wb, hotb);
        }
        ita = na;
        itb = nb;
        CGX_COPY_WORDS(wa, wna);
        CGX_COPY_WORDS(wb, wnb);
        hota = hna;
        hotb = hnb;
        i = in;
      }
    }
  }
}

// CODEC: the wire codec of the compressed items; the FP8 ones exist with KB 8 only, in translation
// units of their own (sra_fp8_*.cu)
template <typename T, int KB, int GPL, int CODEC = kMaxMin>
__global__ void __launch_bounds__(kSraThreads, kSraCtasPerSm) sra_kernel(const __grid_constant__ SraParams p) {
  static_assert(CODEC == kMaxMin || KB == 8, "the FP8 codecs use 8-bit records");
  __shared__ LaneItems li;
  __shared__ int s_abort;
  const int lane = blockIdx.x;
  const uint32_t epoch = *reinterpret_cast<volatile uint32_t*>(&p.sync->epoch) + 1u;
  const int stages = p.stages;
  if (threadIdx.x == 0) s_abort = 0;
  lane_items_load(li, p, p.world, stages);
  trace_mark(p, lane, 0, true);

  _Pragma("unroll 1") for (int t = 0; t < stages; ++t) {
    sra_phase_a<T, KB, GPL, CODEC>(p, li, epoch, t);
    __syncthreads();
    trace_mark(p, lane, 1);
    if (threadIdx.x < 32) {
      signal_peers(p.flags1, p.world, p.rank, p.flag_stride, lane, flag_value(epoch, t));
      trace_mark(p, lane, 6);
    }
  }

  _Pragma("unroll 1") for (int t = 0; t < stages; ++t) {
    if (threadIdx.x < 32 && li.pre[t * p.world + 1] > li.pre[t * p.world]) {
      if (!wait_peers(p.flags1[p.rank], p, lane, flag_value(epoch, t), kSraTimeoutPhase1)) s_abort = 1;
    }
    __syncthreads();
    trace_mark(p, lane, 2);
    if (!s_abort) sra_phase_b<T, KB, GPL, CODEC>(p, li, epoch, t);
    __syncthreads();
    trace_mark(p, lane, 3);
    if (threadIdx.x < 32 && !s_abort) {
      signal_peers(p.flags2, p.world, p.rank, p.flag_stride, lane, flag_value(epoch, t));
      trace_mark(p, lane, 7);
    }
  }

  if (!s_abort) sra_phase_c<T, KB, GPL, false, CODEC>(p, li, epoch, stages);
  trace_mark(p, lane, 5);
  sync_finish(p.sync, epoch, p.lanes);
}

// ===========================================================================
// One-shot allreduce for small / latency-bound messages: ONE signalling hop.
// Every rank quantizes its WHOLE buffer once and stores the packed image into slot `rank` of
// every rank's one-shot region (one multimem.st with NVLS); after one flag exchange every rank
// decodes all W images in rank order and sums them in fp32. Replicas are bit-identical (same
// bytes, same order) and each contribution is quantized exactly once. Costs W/2 x the wire bytes
// of SRA, irrelevant below ~1 MB where latency dominates. (SURVEY.md build plan step 5; replaces
// the reference's tiny-tensor all-to-all, /root/reference/src/common/reducer.cc:35-94.)
// Consecutive calls alternate between two regions (epoch parity): a peer can be one call ahead.
// ===========================================================================
// CODEC as in sra_kernel: an FP8 image holds the codes of x * prescale, and phase 2 sums every
// image's decoded values from +0 in rank order.
template <typename T, int KB, int GPL, int CODEC = kMaxMin>
__global__ void __launch_bounds__(kSraThreads, kSraCtasPerSm) oneshot_kernel(const __grid_constant__ SraParams p) {
  static_assert(CODEC == kMaxMin || KB == 8, "the FP8 codecs use 8-bit records");
  __shared__ LaneItems li;
  __shared__ int s_abort;
  const int lane = blockIdx.x;
  const int r = p.rank, W = p.world;
  const uint32_t warp = threadIdx.x >> 5;
  T* data = reinterpret_cast<T*>(p.data);
  const uint32_t epoch = *reinterpret_cast<volatile uint32_t*>(&p.sync->epoch) + 1u;
  RngKey rng = p.rng;
  rng.seq += epoch - p.epoch_hint;
  rng.stream = (uint32_t)r * 2u;
  if (threadIdx.x == 0) s_abort = 0;
  lane_items_load(li, p, 1, 1);
  trace_mark(p, lane, 0, true);
  const uint32_t region = (epoch & 1u) * p.os_parity_stride;
  const uint32_t total = li.pre[1];
  const SrcSet no_src{nullptr, 0u, 0, -1};

  // ---- phase 1: my image -> slot r of every rank (mine included)
  {
    // with NVLS the switch also delivers my own replica, but asynchronously: my slot is
    // additionally written with a plain local store so that phase 2 never depends on the loopback
    const MultiDst ds{p.recv1, p.mc_recv1, region + (uint32_t)r * p.slot_bytes, W, p.mc_recv1 ? r : -1,
                      p.mc_recv1 ? p.recv1[r] : nullptr};
    for (uint32_t i = warp; i < total; i += kSraWarps) {
      WarpItem it;
      int cs = 0, hot = 0;
      float x[GPL][8];
      fetch_values<T, GPL>(li, p, i, total, it, cs, hot, x);
      if (i + kSraWarps < total) slice_prefetch_l2<T, GPL>(data + lane_item(li, p, i + kSraWarps, 0).elem_off);
      const uint32_t kind = item_kind(it);
      T* blk = data + it.elem_off;
      if constexpr (CODEC != kMaxMin) {
        if (hot == 1) {
          slice_scale<GPL>(x, p.prescale);
          full_send_fp8_x<CODEC, GPL>(x, it, rng, ds);
          continue;
        }
        if (kind == kItemFull) {
          full_send_fp8_scaled_unaligned<T, T, CODEC, GPL, false>(blk, it, p.prescale, rng, ds, (T*)nullptr);
          continue;
        }
        if (kind == kItemBucket) {
          bucket_send_fp8<T, T, CODEC>(blk, it, p.prescale, rng, ds, (T*)nullptr);
          continue;
        }
      }
      if (hot == 1)
        full_send_x<T, KB, GPL, false, true>(x, it, p.prescale, rng, ds, (T*)nullptr);
      else if (hot == 2)
        raw_full_x<T, 0, GPL>(x, blk, it, p.prescale, no_src, ds);
      else if (kind == kItemFull)
        full_send_unaligned<T, T, KB, GPL, false>(blk, it, p.prescale, rng, ds, (T*)nullptr);
      else if (kind == kItemBucket)
        bucket_quantize<T, T>(blk, it, p.prescale, rng, no_src, ds, (T*)nullptr);
      else
        raw_generic<T>(blk, it, p.prescale, no_src, ds, 0);
    }
    __syncthreads();
    if (warp == 0) signal_peers(p.flags1, W, r, p.flag_stride, lane, flag_value(epoch, 0));
  }
  trace_mark(p, lane, 1);

  // ---- phase 2: all W images (mine was written by this CTA, ordered by the bar.sync above)
  {
    if (warp == 0 && total > 0) {
      if (!wait_peers(p.flags1[r], p, lane, flag_value(epoch, 0), kSraTimeoutPhase1)) s_abort = 1;
    }
    __syncthreads();
    trace_mark(p, lane, 2);
    if (!s_abort) {
      const SrcSet ss{p.recv1[r] + region, p.slot_bytes, W, -1};
      const OneDst none{nullptr};
      for (uint32_t i = warp; i < total; i += kSraWarps) {
        const WarpItem it = lane_item(li, p, i, 0);
        const uint32_t kind = item_kind(it);
        T* blk = data + it.elem_off;
        const bool al = group_aligned<T>(blk);
        if constexpr (CODEC != kMaxMin) {
          if (kind == kItemFull) {
            if (al)
              full_recv_sum_fp8<T, CODEC, GPL, true>(ss, it, blk);
            else
              full_recv_sum_fp8_unaligned<T, CODEC, GPL>(ss, it, blk);
            continue;
          }
          if (kind == kItemBucket) {
            bucket_recv_sum_fp8<T, CODEC>(ss, it, blk);
            continue;
          }
        }
        if (kind == kItemFull && al) {
          full_recv_sum<T, KB, GPL, true>(ss, it, blk);
        } else if (kind == kItemFull) {
          full_recv_unaligned<T, KB, GPL>(ss, it, blk);
        } else if (kind == kItemRaw && al) {
          float x[2][8];
          raw_full_x<T, 2, 2>(x, blk, it, 1.0f, ss, none);
        } else if (kind == kItemBucket) {
          bucket_recv<T>(ss, it, blk);
        } else {
          raw_generic<T>(blk, it, 1.0f, ss, none, 2);
        }
      }
    }
  }
  trace_mark(p, lane, 5);
  sync_finish(p.sync, epoch, p.lanes);
}

// ===========================================================================
// Compressed reduce-scatter: phase A of the SRA (every peer's chunk quantized once and pushed into
// its owner's recv1 slot), then a phase B that adds the W-1 decoded copies to my own unquantized
// values in fp32 and stores T(sum) to the output shard. No requantization, no phase C.
// The plan is the shard's layer table replicated W times at stride S (chunk c == copy c), so an
// item of my chunk at element e of the input lands on out[e - rank * S] (p.out_shift).
// Without phase C nothing proves that the peers are done reading my recv1 stores, so the kernel
// ends with a handshake on flags2 (docs/MEMORY_MODEL.md): a peer's next call can only overwrite
// the slots after every lane of this call has finished its reads.
// ===========================================================================
template <typename T, int KB, int GPL, int CODEC = kMaxMin>
__device__ __forceinline__ void rs_phase_b(const SraParams& p, const LaneItems& li) {
  const int r = p.rank, W = p.world;
  const uint32_t warp = threadIdx.x >> 5;
  const T* data = reinterpret_cast<const T*>(p.data);
  T* out = reinterpret_cast<T*>(p.out);
  const SrcSet ss{p.recv1[r], p.slot_bytes, W, r};
  const OneDst none{nullptr};
  const uint32_t end = li.pre[1];
  for (uint32_t i = li.pre[0] + warp; i < end; i += kSraWarps) {
    const WarpItem it = lane_item(li, p, i, 0);
    const uint32_t kind = item_kind(it);
    const T* src = data + it.elem_off;
    T* dst = out + ((uint64_t)it.elem_off - p.out_shift);
    const bool al = group_aligned<T>(src) && group_aligned<T>(dst);
    float x[GPL][8];
    if (al && kind == kItemFull) slice_load_vec<T, GPL>(src, x);
    if (al && kind == kItemRaw) raw_load_vec<T, GPL>(src, x);
    if (i + kSraWarps < end) slice_prefetch_l2<T, GPL>(data + lane_item(li, p, i + kSraWarps, 0).elem_off);
    if (CODEC != kMaxMin && kind == kItemFull) {
      if (al)
        full_rs_fp8_x<T, CODEC, GPL, true>(x, it, p.prescale, ss, dst);
      else
        full_rs_fp8_unaligned<T, CODEC, GPL>(src, it, p.prescale, ss, dst);
    } else if (CODEC != kMaxMin && kind == kItemBucket) {
      bucket_rs_fp8<T, CODEC>(src, it, p.prescale, ss, dst);
    } else if (kind == kItemFull) {
      if (al)
        full_rs_x<T, KB, GPL, true>(x, it, p.prescale, ss, dst);
      else
        full_rs_unaligned<T, KB, GPL>(src, it, p.prescale, ss, dst);
    } else if (kind == kItemBucket) {
      bucket_rs<T>(src, it, p.prescale, ss, dst);
    } else if (kind == kItemRaw && al) {
      raw_full_x<T, 3, GPL>(x, dst, it, p.prescale, ss, none);
    } else {
      raw_rs_generic<T>(src, it, p.prescale, ss, dst);
    }
  }
}

// CODEC: the wire codec of the compressed items; the FP8 ones exist with KB 8 only.
template <typename T, int KB, int GPL, int CODEC = kMaxMin>
__global__ void __launch_bounds__(kSraThreads, kSraCtasPerSm) rs_kernel(const __grid_constant__ SraParams p) {
  static_assert(CODEC == kMaxMin || KB == 8, "the FP8 codecs use 8-bit records");
  __shared__ LaneItems li;
  __shared__ int s_abort;
  const int lane = blockIdx.x;
  const uint32_t epoch = *reinterpret_cast<volatile uint32_t*>(&p.sync->epoch) + 1u;
  const uint32_t flag = flag_value(epoch, 0);
  if (threadIdx.x == 0) s_abort = 0;
  lane_items_load(li, p, p.world, 1);
  trace_mark(p, lane, 0, true);

  sra_phase_a<T, KB, GPL, CODEC>(p, li, epoch, 0);
  __syncthreads();
  trace_mark(p, lane, 1);
  if (threadIdx.x < 32) {
    signal_peers(p.flags1, p.world, p.rank, p.flag_stride, lane, flag);
    if (li.pre[1] > li.pre[0] && !wait_peers(p.flags1[p.rank], p, lane, flag, kSraTimeoutPhase1)) s_abort = 1;
  }
  __syncthreads();
  trace_mark(p, lane, 2);
  if (!s_abort) rs_phase_b<T, KB, GPL, CODEC>(p, li);
  __syncthreads();
  trace_mark(p, lane, 3);

  // slot handshake: every lane, whether or not it had items (a peer's next call may give this
  // lane's slot range to another lane)
  if (threadIdx.x < 32 && !s_abort) {
    signal_peers(p.flags2, p.world, p.rank, p.flag_stride, lane, flag);
    wait_peers(p.flags2[p.rank], p, lane, flag, kSraTimeoutPhase2);
  }
  trace_mark(p, lane, 5);
  sync_finish(p.sync, epoch, p.lanes);
}

// ===========================================================================
// Compressed all-gather: every rank quantizes its own shard once, publishes the record into slot
// `rank` of every peer's recv1 (one multimem.st with NVLS, W-1 peer stores otherwise) and writes
// the self-decoded values to its own chunk of the output; then phase C decodes the peers' chunks
// from recv1, in order of arrival. Every rank's output is the same bytes: decode(Q(in_q)) for
// every q, the owner's chunk included.
// The plan is the shard's layer table replicated W times at stride S (chunk c == copy c): an item
// of my chunk at element e reads in[e - rank * S] (p.out_shift) and writes out[e].
// Like rs_kernel it ends with a handshake on flags2: a peer's next call can only overwrite my
// recv1 slots after every lane of this call has decoded them (docs/MEMORY_MODEL.md).
// CODES (an FP8 codec, p.out_scales set; every item compressed): `out` holds one code byte per
// element and every chunk's records are handed over undecoded; the owner's encoder stores each byte
// it publishes to its own codes and scales too (TeeDst), phase C unpacks the peers' records.
// ===========================================================================
template <typename T, int KB, int GPL, int CODEC = kMaxMin, bool CODES = false>
__device__ __forceinline__ void ag_publish(const SraParams& p, const LaneItems& li, uint32_t epoch) {
  const int r = p.rank, W = p.world;
  const uint32_t warp = threadIdx.x >> 5;
  const T* in = reinterpret_cast<const T*>(p.data);
  T* out = reinterpret_cast<T*>(p.out);
  const RngKey rng = phase_rng(p, epoch, 1u);  // the SRA's publish stream
  const SrcSet no_src{nullptr, 0u, 0, -1};
  // my own slot is skipped by the unicast stores; the multicast also lands there, and nobody reads it
  const MultiDst ds{p.recv1, p.mc_recv1, (uint32_t)r * p.slot_bytes, W, r, nullptr};
  const uint32_t end = li.pre[1];
  // `in` is either disjoint from `out` or exactly its chunk r (then src == dst): every lane loads
  // the elements it later stores itself, before it stores them
  for (uint32_t i = li.pre[0] + warp; i < end; i += kSraWarps) {
    const WarpItem it = lane_item(li, p, i, 0);
    const uint32_t kind = item_kind(it);
    const T* src = in + ((uint64_t)it.elem_off - p.out_shift);
    T* dst = out + it.elem_off;
    const bool al = group_aligned<T>(src) && (CODES || group_aligned<T>(dst));
    float x[GPL][8];
    if (al && kind == kItemFull) slice_load_vec<T, GPL>(src, x);
    if (al && kind == kItemRaw) raw_load_vec<T, GPL>(src, x);
    if (i + kSraWarps < end)
      slice_prefetch_l2<T, GPL>(in + ((uint64_t)lane_item(li, p, i + kSraWarps, 0).elem_off - p.out_shift));
    if constexpr (CODES) {
      const TeeDst<MultiDst> td{ds, CodesDst{reinterpret_cast<uint8_t*>(p.out) + it.elem_off,
                                             p.out_scales + it.elem_off / p.out_bucket, it.meta_off, it.pay_off,
                                             item_n(it)}};
      if (kind == kItemFull && al) {
        slice_scale<GPL>(x, p.prescale);
        full_send_fp8_x<CODEC, GPL>(x, it, rng, td);
      } else if (kind == kItemFull) {
        full_send_fp8_scaled_unaligned<T, T, CODEC, GPL, false>(src, it, p.prescale, rng, td, (T*)nullptr);
      } else {
        bucket_send_fp8<T, T, CODEC>(src, it, p.prescale, rng, td, (T*)nullptr);
      }
      continue;
    }
    if (CODEC != kMaxMin && kind == kItemFull) {
      if (al) {
        slice_scale<GPL>(x, p.prescale);
        full_publish_fp8_x<T, CODEC, GPL, true>(x, it, rng, ds, dst);
      } else {
        full_send_fp8_scaled_unaligned<T, T, CODEC, GPL, true>(src, it, p.prescale, rng, ds, dst);
      }
    } else if (CODEC != kMaxMin && kind == kItemBucket) {
      bucket_send_fp8<T, T, CODEC>(src, it, p.prescale, rng, ds, dst);
    } else if (kind == kItemFull) {
      if (al)
        full_send_x<T, KB, GPL, true, true>(x, it, p.prescale, rng, ds, dst);
      else
        full_send_unaligned<T, T, KB, GPL, true>(src, it, p.prescale, rng, ds, dst);
    } else if (kind == kItemBucket) {
      bucket_quantize<T, T>(src, it, p.prescale, rng, no_src, ds, dst);
    } else if (kind == kItemRaw && al) {
      raw_full_x<T, 0, GPL>(x, dst, it, p.prescale, no_src, ds);
      raw_store_vec<T, GPL>(dst, x);
    } else {
      raw_ag_generic<T>(src, it, p.prescale, ds, dst);
    }
  }
}

template <typename T, int KB, int GPL, int CODEC = kMaxMin, bool CODES = false>
__global__ void __launch_bounds__(kSraThreads, kSraCtasPerSm) ag_kernel(const __grid_constant__ SraParams p) {
  static_assert(CODEC == kMaxMin || KB == 8, "the FP8 codecs use 8-bit records");
  static_assert(!CODES || CODEC != kMaxMin, "codes are delivered for the FP8 codecs only");
  __shared__ LaneItems li;
  __shared__ int s_abort;
  const int lane = blockIdx.x;
  const uint32_t epoch = *reinterpret_cast<volatile uint32_t*>(&p.sync->epoch) + 1u;
  const uint32_t flag = flag_value(epoch, 0);
  if (threadIdx.x == 0) s_abort = 0;
  lane_items_load(li, p, p.world, 1);
  trace_mark(p, lane, 0, true);

  ag_publish<T, KB, GPL, CODEC, CODES>(p, li, epoch);
  __syncthreads();
  trace_mark(p, lane, 3);
  if (threadIdx.x < 32) signal_peers(p.flags1, p.world, p.rank, p.flag_stride, lane, flag);
  sra_phase_c<T, KB, GPL, true, CODEC, CODES>(p, li, epoch, 1, &s_abort);
  __syncthreads();

  // slot handshake, as in rs_kernel: every lane, whether or not it had items
  if (threadIdx.x < 32 && !s_abort) {
    signal_peers(p.flags2, p.world, p.rank, p.flag_stride, lane, flag);
    wait_peers(p.flags2[p.rank], p, lane, flag, kSraTimeoutPhase2);
  }
  trace_mark(p, lane, 5);
  sync_finish(p.sync, epoch, p.lanes);
}

}  // namespace dev

// ---- host side: pick the instantiation --------------------------------------------------
// OP: kOpAllreduce (SRA / one-shot by p.oneshot), kOpReduceScatter or kOpAllGather. The reduce-
// scatter and all-gather kernels are instantiated in translation units of their own
// (rs_* / ag_{f32,f16,bf16}.cu): out-of-line helpers are register-allocated per module, and sharing
// them with another kernel would change the allreduce kernels' spill counts. For the same reason the
// FP8 allreduce (launch_sra_fp8_t: sra_kernel / oneshot_kernel with an FP8 codec) has its own
// sra_fp8_{f32,f16,bf16}.cu.
enum : int { kOpAllreduce = 0, kOpReduceScatter = 1, kOpAllGather = 2 };

template <typename T, int KB, int GPL, int OP, int CODEC = kMaxMin, bool CODES = false>
cudaError_t launch_sra_inst(const SraParams& p, cudaStream_t stream) {
  if constexpr (OP == kOpReduceScatter)
    dev::rs_kernel<T, KB, GPL, CODEC><<<p.lanes, kSraThreads, 0, stream>>>(p);
  else if constexpr (OP == kOpAllGather)
    dev::ag_kernel<T, KB, GPL, CODEC, CODES><<<p.lanes, kSraThreads, 0, stream>>>(p);
  else if (p.oneshot)
    dev::oneshot_kernel<T, KB, GPL, CODEC><<<p.lanes, kSraThreads, 0, stream>>>(p);
  else
    dev::sra_kernel<T, KB, GPL, CODEC><<<p.lanes, kSraThreads, 0, stream>>>(p);
  return cudaGetLastError();
}

template <typename T, int GPL, int OP>
cudaError_t launch_sra_gpl(const SraParams& p, cudaStream_t stream) {
  if (p.codec != kMaxMin) {  // FP8: the reduce-scatter and all-gather of 8-bit plans (the allreduce: launch_sra_fp8_t)
    if constexpr (OP == kOpAllreduce) {
      return cudaErrorInvalidValue;
    } else {
      if (p.uniform_bits != 8) return cudaErrorInvalidValue;
      if constexpr (OP == kOpAllGather) {
        if (p.out_scales != nullptr) {  // the codes output
          if (p.out_bucket == 0) return cudaErrorInvalidValue;
          return dispatch_fp8(p.codec, cudaErrorInvalidValue, [&](auto c) {
            return launch_sra_inst<T, 8, GPL, OP, decltype(c)::value, true>(p, stream);
          });
        }
      }
      if (p.out_scales != nullptr) return cudaErrorInvalidValue;
      return dispatch_fp8(p.codec, cudaErrorInvalidValue,
                          [&](auto c) { return launch_sra_inst<T, 8, GPL, OP, decltype(c)::value>(p, stream); });
    }
  }
  if (p.out_scales != nullptr) return cudaErrorInvalidValue;
  switch (p.uniform_bits) {
    case 2: return launch_sra_inst<T, 2, GPL, OP>(p, stream);
    case 4: return launch_sra_inst<T, 4, GPL, OP>(p, stream);
    case 8: return launch_sra_inst<T, 8, GPL, OP>(p, stream);
    default: return launch_sra_inst<T, 0, GPL, OP>(p, stream);
  }
}

template <typename T, int OP = kOpAllreduce>
cudaError_t launch_sra_t(const SraParams& p, cudaStream_t stream) {
  return p.slice_elems == 1024 ? launch_sra_gpl<T, 4, OP>(p, stream) : launch_sra_gpl<T, 2, OP>(p, stream);
}

// The FP8 allreduce: sra_kernel / oneshot_kernel of an 8-bit plan with an FP8 p.codec
template <typename T, int GPL>
cudaError_t launch_sra_fp8_gpl(const SraParams& p, cudaStream_t stream) {
  if (p.uniform_bits != 8) return cudaErrorInvalidValue;
  return dispatch_fp8(p.codec, cudaErrorInvalidValue,
                      [&](auto c) { return launch_sra_inst<T, 8, GPL, kOpAllreduce, decltype(c)::value>(p, stream); });
}
template <typename T>
cudaError_t launch_sra_fp8_t(const SraParams& p, cudaStream_t stream) {
  return p.slice_elems == 1024 ? launch_sra_fp8_gpl<T, 4>(p, stream) : launch_sra_fp8_gpl<T, 2>(p, stream);
}

template <typename T>
int sra_resident_per_sm_t() {
  int a = 0, b = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, dev::sra_kernel<T, 0, 2>, kSraThreads, 0) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, dev::sra_kernel<T, 0, 4>, kSraThreads, 0) != cudaSuccess)
    return 0;
  return a < b ? a : b;
}

// defined once per dtype in sra_{f32,f16,bf16}.cu
cudaError_t launch_sra_f32(const SraParams& p, cudaStream_t stream);
cudaError_t launch_sra_f16(const SraParams& p, cudaStream_t stream);
cudaError_t launch_sra_bf16(const SraParams& p, cudaStream_t stream);
int sra_resident_per_sm_f32();
int sra_resident_per_sm_f16();
int sra_resident_per_sm_bf16();
// defined once per dtype in rs_{f32,f16,bf16}.cu
cudaError_t launch_rs_f32(const SraParams& p, cudaStream_t stream);
cudaError_t launch_rs_f16(const SraParams& p, cudaStream_t stream);
cudaError_t launch_rs_bf16(const SraParams& p, cudaStream_t stream);
// defined once per dtype in ag_{f32,f16,bf16}.cu
cudaError_t launch_ag_f32(const SraParams& p, cudaStream_t stream);
cudaError_t launch_ag_f16(const SraParams& p, cudaStream_t stream);
cudaError_t launch_ag_bf16(const SraParams& p, cudaStream_t stream);
// defined once per dtype in sra_fp8_{f32,f16,bf16}.cu
cudaError_t launch_sra_fp8_f32(const SraParams& p, cudaStream_t stream);
cudaError_t launch_sra_fp8_f16(const SraParams& p, cudaStream_t stream);
cudaError_t launch_sra_fp8_bf16(const SraParams& p, cudaStream_t stream);

}  // namespace cgx

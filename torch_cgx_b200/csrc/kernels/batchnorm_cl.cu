// Training-mode BatchNorm on channels_last input (an [M = N*H*W][C] matrix), forward and backward, with the
// block ReLU optionally fused (the backward section further down).
//
// Bit-identical to ATen's channels_last path (batch_norm_collect_statistics_channels_last_kernel<Var>,
// batch_norm_update_stats_and_invert, batch_norm_transform_input_channels_last_kernel) followed by
// relu_. ATen's result depends only on a fixed order of float operations, not on its memory schedule:
//
//  * (BX, BY, GX, GY) = flexible_launch_configs(M, C, coop = true). A chain (c, by, ty, j), j = 0..3, runs
//    Welford updates over rows m = by*BY + ty + (4i + j)*BY*GY for i = 0 .. L-1, L = 1 + (M-1)/(4*BY*GY),
//    with inv = 1/count correctly rounded. Rows >= M still update, with x = 0, inv = 0 and weight 0:
//    that turns an infinite mean into NaN and an overflowing mean*mean into a NaN m2.
//  * The chains of a thread merge j = 1, 2, 3 into 0, then the ty of a block merge in a halving tree.
//    With GY > 1 the last block merges the staged block results y = ty, ty + BY, ... from the zero
//    state and runs the tree again. Every merge rounds, also one with an empty side.
//  * var = m2/count, running stats r = mean*momentum + (1 - momentum)*r (var scaled by the Bessel factor
//    N/(N-1) computed in double), invstd = rsqrt(var + eps).
//
// The contractions into FMAs are those of ATen's sm_90 SASS. The compiler contracted the two products
// of the merge's mean differently at the two kinds of call site: the per-thread merge of the four
// chains fuses mean_new*count_new, the block and grid merges fuse mean*count. This extension builds
// with --fmad=false and writes every FMA explicitly.
//
// The physical mapping is free and differs: a thread runs one chain for 8 (16-bit) or 4 (fp32)
// channels with 16-byte loads and U rows in flight; a block holds one ATen block row `by` and a slab
// of channels; the chain results meet in shared memory for the merges. Short chains run on 256-thread
// blocks light enough that 3-4 of them share an SM, so one block's merges, fence and arrival run while
// the others' loads are in flight; long chains on 512-thread blocks (chain_launch).
#include "device_utils.cuh"
#include "launch.h"

namespace cgx {
using namespace dev;

namespace {
constexpr int kLongChain = 16;    // chains of more rows run on wide blocks (see chain_launch)
constexpr int block_threads(bool wide) { return wide ? 512 : 256; }
constexpr int kSmemSlots = 4096;  // chains x slab channels; ATen's configs need at most 4096 (see below)
constexpr int kMaxStaged = 8;     // staged rows per slot in the grid merge: GY >= 8 means BY >= 16, GY <= 128

template <typename T, int V>
struct Row {
  static_assert(V == 1 || V * sizeof(T) == 16, "a vector is one element or 16 bytes");
  union {
    uint4 u;
    T e[V];
  } v;
  __device__ __forceinline__ void load(const T* p) {
    if constexpr (V == 1)
      v.e[0] = p[0];
    else
      v.u = __ldg(reinterpret_cast<const uint4*>(p));
  }
  __device__ __forceinline__ void zero() {
    if constexpr (V == 1)
      v.e[0] = DT<T>::from_float(0.0f);
    else
      v.u = make_uint4(0u, 0u, 0u, 0u);
  }
  __device__ __forceinline__ float f(int k) const { return DT<T>::to_float(v.e[k]); }
};

// ATen's welford_merge_element; FUSE_NEW: mean_new*count_new is the contracted product, else mean*count
template <bool FUSE_NEW>
__device__ __forceinline__ void welford_merge(int& n, float& mean, float& m2, int nb, float mb, float m2b) {
  const float fa = (float)n, fb = (float)nb;
  const float factor = __frcp_rn((float)max(1, n + nb));
  const float d = __fadd_rn(mean, -mb);
  const float s = FUSE_NEW ? __fmaf_rn(mb, fb, __fmul_rn(mean, fa)) : __fmaf_rn(mean, fa, __fmul_rn(mb, fb));
  const float t = __fmul_rn(__fmul_rn(__fmul_rn(d, d), fb), fa);
  mean = __fmul_rn(s, factor);
  m2 = __fadd_rn(m2, __fmaf_rn(t, factor, m2b));
  n += nb;
}

// The chain results of a block in dynamic shared memory, sized at its launch (forward_t, backward_t): 4*BY*W
// slots per array. ResNet-50's short-chain blocks need 16.6 KB instead of a fixed 40 KB, so shared memory
// does not limit how many of them share an SM.
extern __shared__ float bn_smem[];

struct Smem {
  float* mean;
  float* m2;
  int* cnt;  // one count per chain: counts do not depend on the channel
  __device__ Smem(int slots) : mean(bn_smem), m2(bn_smem + slots), cnt(reinterpret_cast<int*>(bn_smem + 2 * slots)) {}
};

// halving tree over ty of slot (ty*4) for the W channels of the slab (welford_merge_block_vertical)
__device__ __forceinline__ void vertical_tree(Smem& s, int BY, int W, int wvalid) {
  for (int off = BY / 2; off > 0; off >>= 1) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < off * W; idx += blockDim.x) {
      const int ty = idx / W, cc = idx - ty * W;
      if (cc >= wvalid) continue;
      const int a = ty * 4 * W + cc, b = (ty + off) * 4 * W + cc;
      int n = s.cnt[ty * 4];
      welford_merge<false>(n, s.mean[a], s.m2[a], s.cnt[(ty + off) * 4], s.mean[b], s.m2[b]);
    }
    __syncthreads();
    if ((int)threadIdx.x < off) s.cnt[threadIdx.x * 4] += s.cnt[(threadIdx.x + off) * 4];
  }
  __syncthreads();
}

struct StatsArgs {
  int M, C, BY, GY, L, G;
  float* staging;  // [3][GY][C]: mean, m2, count (int bits); used when GY > 1
  int* sem;        // one self-resetting arrival counter per slab
  float *save_mean, *save_invstd, *run_mean, *run_var;
  float momentum, bessel, eps;
};

// U = 4 rows in flight for chains of at most 4 rows (fits four 256-thread blocks per SM), else 8 (three)
template <typename T, int V, int U, bool WIDE>
__global__ void __launch_bounds__(block_threads(WIDE), WIDE ? 1 : (U == 4 ? 4 : 3))
bn_stats_kernel(const T* __restrict__ x, const StatsArgs a) {
  const int G = a.G, W = G * V, by = blockIdx.y;
  const int c0 = blockIdx.x * W;
  const int wvalid = min(W, a.C - c0);
  const int nch = a.BY * 4;
  Smem s(nch * W);
  __shared__ bool last;
  const int g = threadIdx.x % G;
  const int c = c0 + g * V;
  const int rstride = a.BY * a.GY;  // rows between a chain's consecutive (4i + j)

  // ---- chains: Welford over rows, U rows in flight
  for (int ch = threadIdx.x / G; ch < nch; ch += blockDim.x / G) {
    const int ty = ch >> 2, j = ch & 3;
    const int m0 = by * a.BY + ty;
    float mean[V], m2[V];
#pragma unroll
    for (int k = 0; k < V; ++k) mean[k] = m2[k] = 0.0f;
    int cnt = 0;
    if (c < a.C) {
      for (int i0 = 0; i0 < a.L; i0 += U) {
        Row<T, V> r[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t m = (int64_t)m0 + (int64_t)(4 * (i0 + u) + j) * rstride;
          if (i0 + u < a.L && m < a.M)
            r[u].load(x + m * a.C + c);
          else
            r[u].zero();
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (i0 + u >= a.L) break;
          const int64_t m = (int64_t)m0 + (int64_t)(4 * (i0 + u) + j) * rstride;
          const bool valid = m < a.M;
          float inv = 0.0f, w = 0.0f;
          if (valid) {
            ++cnt;
            inv = __frcp_rn((float)cnt);
            w = 1.0f;
          }
#pragma unroll
          for (int k = 0; k < V; ++k) {
            const float xv = r[u].f(k);
            const float d0 = __fadd_rn(xv, -mean[k]);
            mean[k] = __fmaf_rn(d0, inv, mean[k]);
            const float d1 = __fadd_rn(xv, -mean[k]);
            m2[k] = __fmaf_rn(__fmul_rn(d0, d1), w, m2[k]);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < V; ++k) {
        s.mean[ch * W + g * V + k] = mean[k];
        s.m2[ch * W + g * V + k] = m2[k];
      }
    }
    if (g == 0) s.cnt[ch] = cnt;
  }
  __syncthreads();

  // ---- merge the four chains of each (ty, channel) into j = 0
  for (int idx = threadIdx.x; idx < a.BY * W; idx += blockDim.x) {
    const int ty = idx / W, cc = idx - ty * W;
    if (cc >= wvalid) continue;
    const int b0 = ty * 4;
    int n = s.cnt[b0];
    float mean = s.mean[b0 * W + cc], m2 = s.m2[b0 * W + cc];
#pragma unroll
    for (int jj = 1; jj < 4; ++jj)
      welford_merge<true>(n, mean, m2, s.cnt[b0 + jj], s.mean[(b0 + jj) * W + cc], s.m2[(b0 + jj) * W + cc]);
    s.mean[b0 * W + cc] = mean;
    s.m2[b0 * W + cc] = m2;
  }
  __syncthreads();
  if ((int)threadIdx.x < a.BY) {
    const int b0 = threadIdx.x * 4;
    s.cnt[b0] = s.cnt[b0] + s.cnt[b0 + 1] + s.cnt[b0 + 2] + s.cnt[b0 + 3];
  }
  vertical_tree(s, a.BY, W, wvalid);

  if (a.GY > 1) {
    const size_t plane = (size_t)a.GY * a.C;
    float* st_mean = a.staging;
    float* st_m2 = a.staging + plane;
    int* st_cnt = reinterpret_cast<int*>(a.staging + 2 * plane);
    for (int cc = threadIdx.x; cc < wvalid; cc += blockDim.x) {
      const size_t o = (size_t)by * a.C + c0 + cc;
      st_mean[o] = s.mean[cc];
      st_m2[o] = s.m2[cc];
      st_cnt[o] = s.cnt[0];
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const int old = atomicAdd(&a.sem[blockIdx.x], 1);
      last = old == a.GY - 1;
      if (last) a.sem[blockIdx.x] = 0;  // ready for the next launch on this stream
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // the last block: slot ty*4 merges staged rows y = ty, ty + BY, ... starting from the zero state;
    // all of a slot's staged loads are issued before its first merge
    for (int idx = threadIdx.x; idx < a.BY * W; idx += blockDim.x) {
      const int ty = idx / W, cc = idx - ty * W;
      if (cc >= wvalid) continue;
      int nb[kMaxStaged];
      float mb[kMaxStaged], m2b[kMaxStaged];
#pragma unroll
      for (int k = 0; k < kMaxStaged; ++k) {
        const int y = ty + k * a.BY;
        nb[k] = 0;
        mb[k] = m2b[k] = 0.0f;
        if (y < a.GY) {
          const size_t o = (size_t)y * a.C + c0 + cc;
          nb[k] = __ldcg(st_cnt + o);
          mb[k] = __ldcg(st_mean + o);
          m2b[k] = __ldcg(st_m2 + o);
        }
      }
      int n = 0;
      float mean = 0.0f, m2 = 0.0f;
#pragma unroll
      for (int k = 0; k < kMaxStaged; ++k)
        if (ty + k * a.BY < a.GY) welford_merge<false>(n, mean, m2, nb[k], mb[k], m2b[k]);
      s.mean[ty * 4 * W + cc] = mean;
      s.m2[ty * 4 * W + cc] = m2;
      if (cc == 0) s.cnt[ty * 4] = n;
    }
    vertical_tree(s, a.BY, W, wvalid);
  } else if (by != 0) {
    return;
  }

  // ---- finalize (batch_norm_update_stats_and_invert)
  const float omm = __fadd_rn(1.0f, -a.momentum);
  for (int cc = threadIdx.x; cc < wvalid; cc += blockDim.x) {
    const int ch = c0 + cc;
    const float mean = s.mean[cc];
    const float var = __fdiv_rn(s.m2[cc], (float)s.cnt[0]);
    a.save_mean[ch] = mean;
    a.run_mean[ch] = __fmaf_rn(mean, a.momentum, __fmul_rn(omm, a.run_mean[ch]));
    a.run_var[ch] = __fmaf_rn(__fmul_rn(var, a.bessel), a.momentum, __fmul_rn(omm, a.run_var[ch]));
    a.save_invstd[ch] = rsqrtf(__fadd_rn(var, a.eps));
  }
}

// T(w*(x - mean)*invstd + b), contracted as ATen's transform: fma((x - mean)*w, invstd, b)
template <typename T>
__device__ __forceinline__ T bn_out(float x, float mean, float w, float invstd, float b) {
  return DT<T>::from_float(__fmaf_rn(__fmul_rn(__fadd_rn(x, -mean), w), invstd, b));
}

// y = bn_out; with RELU the eager relu_ on the T value: (y <= 0) ? +0 : y, a NaN kept
template <typename T, int V, bool RELU>
__global__ void __launch_bounds__(256)
bn_transform_kernel(const T* __restrict__ x, T* __restrict__ y, const float* __restrict__ mean,
                    const float* __restrict__ invstd, const float* __restrict__ weight,
                    const float* __restrict__ bias, int M, int C) {
  constexpr int U = 4;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c >= C) return;
  float mu[V], is[V], w[V], b[V];
#pragma unroll
  for (int k = 0; k < V; ++k) {
    mu[k] = mean[c + k];
    is[k] = invstd[c + k];
    w[k] = weight[c + k];
    b[k] = bias[c + k];
  }
  const int rs = gridDim.y * blockDim.y;
  for (int m0 = blockIdx.y * blockDim.y + threadIdx.y; m0 < M; m0 += rs * U) {
    Row<T, V> r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t m = (int64_t)m0 + (int64_t)u * rs;
      if (m < M) r[u].load(x + m * C + c);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t m = (int64_t)m0 + (int64_t)u * rs;
      if (m >= M) break;
      Row<T, V> o;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        T t = bn_out<T>(r[u].f(k), mu[k], w[k], is[k], b[k]);
        if (RELU && DT<T>::to_float(t) <= 0.0f) t = DT<T>::from_float(0.0f);
        o.v.e[k] = t;
      }
      if constexpr (V == 1)
        y[m * C + c] = o.v.e[0];
      else
        *reinterpret_cast<uint4*>(y + m * C + c) = o.v.u;
    }
  }
}

// ---- backward: ATen's batch_norm_backward_reduce_channels_last_kernel and
// batch_norm_backward_elemt_channels_last_kernel (train), with the gradient of an optional ReLU folded in.
// With RELU the incoming gradient is taken as +0 where bn_out(x) <= 0, which is what
// threshold_backward(g, relu_(bn_out), 0) hands the eager backward; the mask comes from x, so y is not read.
//
// The reduction has the statistics kernel's chains and tree with plain fp32 sums. Per row (rows >= M
// with x = g = 0, as ATen): sum_dy += g; sum_dy_xmu = fma(x - mean, g, sum_dy_xmu). Chains merge
// j = 1, 2, 3 into 0 in order, the block tree adds [ty + off] into [ty], the grid merge adds the staged
// block sums y = ty, ty + BY, ... to 0.0f. grad_weight = sum_dy_xmu * invstd, grad_bias = sum_dy.
// The element-wise kernel (ATen's SASS): gx = T(w*invstd * fma(-f1, x - mean, fma(-sum_dy, nf, g))),
// f1 = ((invstd*invstd)*sum_dy_xmu)*nf, nf = float(1.0 / M) computed in double.

template <typename T, int V, bool RELU>
__device__ __forceinline__ float masked_grad(float g, float x, float mu, float w, float is, float b) {
  if (RELU && DT<T>::to_float(bn_out<T>(x, mu, w, is, b)) <= 0.0f) return 0.0f;
  return g;
}

struct SmemSum {  // as Smem
  float* dy;
  float* xmu;
  __device__ SmemSum(int slots) : dy(bn_smem), xmu(bn_smem + slots) {}
};

struct ReduceArgs {
  int M, C, BY, GY, L, G;
  float* staging;  // [2][GY][C]: sum_dy, sum_dy_xmu; used when GY > 1
  int* sem;
  const float *mean, *invstd, *weight, *bias;
  float *sum_dy, *sum_dy_xmu, *grad_weight, *grad_bias;
};

__device__ __forceinline__ void sum_tree(SmemSum& s, int BY, int W, int wvalid) {
  for (int off = BY / 2; off > 0; off >>= 1) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < off * W; idx += blockDim.x) {
      const int ty = idx / W, cc = idx - ty * W;
      if (cc >= wvalid) continue;
      const int a = ty * 4 * W + cc, b = (ty + off) * 4 * W + cc;
      s.dy[a] = __fadd_rn(s.dy[a], s.dy[b]);
      s.xmu[a] = __fadd_rn(s.xmu[a], s.xmu[b]);
    }
  }
  __syncthreads();
}

// MASK_SMEM (with RELU, on 256-thread blocks): the mask's invstd, weight and bias come from shared memory,
// which fits three blocks per SM instead of two
template <typename T, int V, bool RELU, bool WIDE, bool MASK_SMEM>
__global__ void __launch_bounds__(block_threads(WIDE), WIDE ? 1 : (RELU && !MASK_SMEM ? 2 : 3))
bn_bwd_reduce_kernel(const T* __restrict__ gy, const T* __restrict__ x, const ReduceArgs a) {
  constexpr int U = 4;  // rows of one chain in flight per thread, for each of g and x
  const int G = a.G, W = G * V, by = blockIdx.y;
  const int c0 = blockIdx.x * W;
  const int wvalid = min(W, a.C - c0);
  const int nch = a.BY * 4;
  SmemSum s(nch * W);
  __shared__ bool last;
  const int g = threadIdx.x % G;
  const int c = c0 + g * V;
  const int rstride = a.BY * a.GY;

  // read at every use (volatile, so they are not hoisted into registers)
  constexpr bool kMaskSmem = RELU && MASK_SMEM;
  float* const prm = bn_smem + 2 * nch * W;  // [3][W]
  if (kMaskSmem) {
    for (int cc = threadIdx.x; cc < wvalid; cc += blockDim.x) {
      prm[cc] = a.invstd[c0 + cc];
      prm[W + cc] = a.weight[c0 + cc];
      prm[2 * W + cc] = a.bias[c0 + cc];
    }
    __syncthreads();
  }
  if (c < a.C) {
    float mu[V], is[V], w[V], b[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      mu[k] = a.mean[c + k];
      is[k] = RELU && !kMaskSmem ? a.invstd[c + k] : 0.0f;
      w[k] = RELU && !kMaskSmem ? a.weight[c + k] : 0.0f;
      b[k] = RELU && !kMaskSmem ? a.bias[c + k] : 0.0f;
    }
    for (int ch = threadIdx.x / G; ch < nch; ch += blockDim.x / G) {
      const int ty = ch >> 2, j = ch & 3;
      const int m0 = by * a.BY + ty;
      float sdy[V], sxmu[V];
#pragma unroll
      for (int k = 0; k < V; ++k) sdy[k] = sxmu[k] = 0.0f;
      for (int i0 = 0; i0 < a.L; i0 += U) {
        Row<T, V> rg[U], rx[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t m = (int64_t)m0 + (int64_t)(4 * (i0 + u) + j) * rstride;
          if (i0 + u < a.L && m < a.M) {
            rg[u].load(gy + m * a.C + c);
            rx[u].load(x + m * a.C + c);
          } else {
            rg[u].zero();
            rx[u].zero();
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (i0 + u >= a.L) break;
#pragma unroll
          for (int k = 0; k < V; ++k) {
            const float xv = rx[u].f(k);
            float isk = is[k], wk = w[k], bk = b[k];
            if (kMaskSmem) {
              const volatile float* p = prm + g * V + k;
              isk = p[0];
              wk = p[W];
              bk = p[2 * W];
            }
            const float gv = masked_grad<T, V, RELU>(rg[u].f(k), xv, mu[k], wk, isk, bk);
            sdy[k] = __fadd_rn(sdy[k], gv);
            sxmu[k] = __fmaf_rn(__fadd_rn(xv, -mu[k]), gv, sxmu[k]);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < V; ++k) {
        s.dy[ch * W + g * V + k] = sdy[k];
        s.xmu[ch * W + g * V + k] = sxmu[k];
      }
    }
  }
  __syncthreads();

  for (int idx = threadIdx.x; idx < a.BY * W; idx += blockDim.x) {
    const int ty = idx / W, cc = idx - ty * W;
    if (cc >= wvalid) continue;
    const int o = ty * 4 * W + cc;
    float dy = s.dy[o], xmu = s.xmu[o];
#pragma unroll
    for (int jj = 1; jj < 4; ++jj) {
      dy = __fadd_rn(dy, s.dy[o + jj * W]);
      xmu = __fadd_rn(xmu, s.xmu[o + jj * W]);
    }
    s.dy[o] = dy;
    s.xmu[o] = xmu;
  }
  sum_tree(s, a.BY, W, wvalid);

  if (a.GY > 1) {
    const size_t plane = (size_t)a.GY * a.C;
    float* st_dy = a.staging;
    float* st_xmu = a.staging + plane;
    for (int cc = threadIdx.x; cc < wvalid; cc += blockDim.x) {
      const size_t o = (size_t)by * a.C + c0 + cc;
      st_dy[o] = s.dy[cc];
      st_xmu[o] = s.xmu[cc];
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const int old = atomicAdd(&a.sem[blockIdx.x], 1);
      last = old == a.GY - 1;
      if (last) a.sem[blockIdx.x] = 0;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    for (int idx = threadIdx.x; idx < a.BY * W; idx += blockDim.x) {
      const int ty = idx / W, cc = idx - ty * W;
      if (cc >= wvalid) continue;
      float bdy[kMaxStaged], bxmu[kMaxStaged];
#pragma unroll
      for (int k = 0; k < kMaxStaged; ++k) {
        const int y = ty + k * a.BY;
        bdy[k] = bxmu[k] = 0.0f;
        if (y < a.GY) {
          const size_t o = (size_t)y * a.C + c0 + cc;
          bdy[k] = __ldcg(st_dy + o);
          bxmu[k] = __ldcg(st_xmu + o);
        }
      }
      float dy = 0.0f, xmu = 0.0f;
#pragma unroll
      for (int k = 0; k < kMaxStaged; ++k) {
        if (ty + k * a.BY < a.GY) {
          dy = __fadd_rn(dy, bdy[k]);
          xmu = __fadd_rn(xmu, bxmu[k]);
        }
      }
      s.dy[ty * 4 * W + cc] = dy;
      s.xmu[ty * 4 * W + cc] = xmu;
    }
    sum_tree(s, a.BY, W, wvalid);
  } else if (by != 0) {
    return;
  }

  for (int cc = threadIdx.x; cc < wvalid; cc += blockDim.x) {
    const int ch = c0 + cc;
    a.sum_dy[ch] = s.dy[cc];
    a.sum_dy_xmu[ch] = s.xmu[cc];
    a.grad_bias[ch] = s.dy[cc];
    a.grad_weight[ch] = __fmul_rn(s.xmu[cc], a.invstd[ch]);
  }
}

template <typename T, int V, bool RELU>
__global__ void __launch_bounds__(256)
bn_bwd_elemt_kernel(const T* __restrict__ gy, const T* __restrict__ x, T* __restrict__ gx,
                    const float* __restrict__ mean, const float* __restrict__ invstd,
                    const float* __restrict__ weight, const float* __restrict__ bias,
                    const float* __restrict__ sum_dy, const float* __restrict__ sum_dy_xmu, float nf, int M,
                    int C) {
  constexpr int U = 4;
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c >= C) return;
  float mu[V], is[V], w[V], b[V], f1[V], f2[V], sdy[V];
#pragma unroll
  for (int k = 0; k < V; ++k) {
    mu[k] = mean[c + k];
    is[k] = invstd[c + k];
    w[k] = weight[c + k];
    b[k] = RELU ? bias[c + k] : 0.0f;
    f1[k] = __fmul_rn(__fmul_rn(__fmul_rn(is[k], is[k]), sum_dy_xmu[c + k]), nf);
    f2[k] = __fmul_rn(is[k], w[k]);
    sdy[k] = sum_dy[c + k];
  }
  const int rs = gridDim.y * blockDim.y;
  for (int m0 = blockIdx.y * blockDim.y + threadIdx.y; m0 < M; m0 += rs * U) {
    Row<T, V> rg[U], rx[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t m = (int64_t)m0 + (int64_t)u * rs;
      if (m < M) {
        rg[u].load(gy + m * C + c);
        rx[u].load(x + m * C + c);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t m = (int64_t)m0 + (int64_t)u * rs;
      if (m >= M) break;
      Row<T, V> o;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float xv = rx[u].f(k);
        const float gv = masked_grad<T, V, RELU>(rg[u].f(k), xv, mu[k], w[k], is[k], b[k]);
        const float t = __fmaf_rn(-f1[k], __fadd_rn(xv, -mu[k]), __fmaf_rn(-sdy[k], nf, gv));
        o.v.e[k] = DT<T>::from_float(__fmul_rn(f2[k], t));
      }
      if constexpr (V == 1)
        gx[m * C + c] = o.v.e[0];
      else
        *reinterpret_cast<uint4*>(gx + m * C + c) = o.v.u;
    }
  }
}

int last_pow2(unsigned n) {  // ATen's lastPow2
  n |= n >> 1;
  n |= n >> 2;
  n |= n >> 4;
  n |= n >> 8;
  n |= n >> 16;
  return std::max<int>(1, (int)(n - (n >> 1)));
}
int ceil_div(int a, int b) { return (a + b - 1) / b; }

struct AtenGrid {
  int by, gy;
};
// ATen's flexible_launch_configs(M, C, coop = true); only BY and GY enter the arithmetic
AtenGrid aten_grid(int M, int C) {
  const int bx = std::min(last_pow2(C), 32);
  const int by = std::min(last_pow2(ceil_div(M, 16)), 512 / bx);
  const int gy = std::min(ceil_div(M, by * 16), 128);
  return {by, gy < 8 ? 1 : gy};
}

// The launch of the two chain kernels: grid (slabs, GY), G vector groups of V channels per slab, and
// threads over (chain, group). Two block shapes, chosen from the chain length L:
//  * short chains (L <= kLongChain; ResNet-50's 28x28 and smaller layers): 256 threads, G <= 4, and three
//    or four blocks per SM, so the merges and arrivals of one block overlap the loads of the others;
//  * long chains (its 56x56 and 112x112 layers): 512 threads, G <= 8, one block per SM. There each block
//    streams long enough that its merges cost little, and smaller blocks measured slower at C >= 128.
// The chain results of a block fit kSmemSlots: a slab holds at most 64 channels (W); with C >= 32,
// BX = 32 so BY <= 16 and 4*BY*W <= 4096; with C < 32, W = C < 2*BX and 4*BY <= 2048/BX.
struct ChainLaunch {
  int by, gy, G, nslab, threads, L;
  int slots;  // chain results per shared array: 4*BY chains x W channels
  bool wide;
};
template <int V>
ChainLaunch chain_launch(int M, int C) {
  const AtenGrid ag = aten_grid(M, C);
  ChainLaunch l;
  l.by = ag.by;
  l.gy = ag.gy;
  l.L = 1 + (M - 1) / (l.by * l.gy * 4);
  l.wide = l.L > kLongChain;
  l.G = std::min(V == 1 ? 32 : (l.wide ? 8 : 4), ceil_div(C, V));
  l.nslab = ceil_div(C, l.G * V);
  l.threads = l.G * std::min(4 * l.by, block_threads(l.wide) / l.G);
  l.slots = 4 * l.by * l.G * V;
  return l;
}

// the bounds the chain kernels rely on: shared-memory slots (so at most 40 KB, below the 48 KB a launch
// may take without opting in) and the staged rows of the grid merge
bool chain_launch_ok(const ChainLaunch& l) {
  return l.slots <= kSmemSlots && (l.gy == 1 || ceil_div(l.gy, l.by) <= kMaxStaged);
}

dim3 elementwise_grid(int M, int C, int V, dim3* block) {
  const int cv = C / V;
  const int tx = std::min(cv, 32), ty = 256 / tx;
  const int gx = ceil_div(cv, tx);
  *block = dim3(tx, ty);
  return dim3(gx, std::max(1, std::min(ceil_div(M, ty * 4), 2048 / gx)));
}

template <typename T, int V>
cudaError_t forward_t(const BnForwardArgs& p, cudaStream_t stream) {
  const int M = p.M, C = p.C;
  const ChainLaunch l = chain_launch<V>(M, C);
  const int by = l.by, gy = l.gy, G = l.G, nslab = l.nslab, threads = l.threads;
  if (!chain_launch_ok(l)) return cudaErrorInvalidConfiguration;
  if (gy > 1 && (p.staging == nullptr || p.sem_len < nslab)) return cudaErrorInvalidValue;

  StatsArgs a;
  a.M = M;
  a.C = C;
  a.BY = by;
  a.GY = gy;
  a.L = l.L;
  a.G = G;
  a.staging = p.staging;
  a.sem = p.sem;
  a.save_mean = p.save_mean;
  a.save_invstd = p.save_invstd;
  a.run_mean = p.running_mean;
  a.run_var = p.running_var;
  a.momentum = (float)p.momentum;
  a.bessel = (float)((double)M / (double)(M - 1));
  a.eps = (float)p.eps;
  const T* x = (const T*)p.x;
  const dim3 grid(nslab, gy);
  const size_t smem = (2 * (size_t)l.slots + 4 * by) * sizeof(float);  // mean, m2, one count per chain
  if (l.wide)
    bn_stats_kernel<T, V, 8, true><<<grid, threads, smem, stream>>>(x, a);
  else if (l.L <= 4)
    bn_stats_kernel<T, V, 4, false><<<grid, threads, smem, stream>>>(x, a);
  else
    bn_stats_kernel<T, V, 8, false><<<grid, threads, smem, stream>>>(x, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;

  dim3 tblock;
  const dim3 tgrid = elementwise_grid(M, C, V, &tblock);
  if (p.relu)
    bn_transform_kernel<T, V, true><<<tgrid, tblock, 0, stream>>>(x, (T*)p.y, p.save_mean, p.save_invstd,
                                                                   p.weight, p.bias, M, C);
  else
    bn_transform_kernel<T, V, false><<<tgrid, tblock, 0, stream>>>(x, (T*)p.y, p.save_mean, p.save_invstd,
                                                                    p.weight, p.bias, M, C);
  return cudaGetLastError();
}

template <typename T, int V, bool RELU>
cudaError_t backward_t(const BnBackwardArgs& p, cudaStream_t stream) {
  const int M = p.M, C = p.C;
  const ChainLaunch l = chain_launch<V>(M, C);
  if (!chain_launch_ok(l)) return cudaErrorInvalidConfiguration;
  if (l.gy > 1 && (p.staging == nullptr || p.sem_len < l.nslab)) return cudaErrorInvalidValue;
  ReduceArgs a;
  a.M = M;
  a.C = C;
  a.BY = l.by;
  a.GY = l.gy;
  a.L = l.L;
  a.G = l.G;
  a.staging = p.staging;
  a.sem = p.sem;
  a.mean = p.mean;
  a.invstd = p.invstd;
  a.weight = p.weight;
  a.bias = p.bias;
  a.sum_dy = p.sum_dy;
  a.sum_dy_xmu = p.sum_dy_xmu;
  a.grad_weight = p.grad_weight;
  a.grad_bias = p.grad_bias;
  const T* g = (const T*)p.g;
  const T* x = (const T*)p.x;
  // sum_dy, sum_dy_xmu; on 256-thread blocks with the mask also its invstd, weight and bias per channel
  // The mask from shared memory pays for its extra loads only where blocks are short-lived (L <= 4: the
  // 14x14 and 7x7 layers); it measured slower at 28x28.
  const bool mask_smem = RELU && !l.wide && l.L <= 4;
  const size_t smem = (2 * (size_t)l.slots + (mask_smem ? 3 * l.G * V : 0)) * sizeof(float);
  const dim3 rgrid(l.nslab, l.gy);
  if (l.wide)
    bn_bwd_reduce_kernel<T, V, RELU, true, false><<<rgrid, l.threads, smem, stream>>>(g, x, a);
  else if (mask_smem)
    bn_bwd_reduce_kernel<T, V, RELU, false, RELU><<<rgrid, l.threads, smem, stream>>>(g, x, a);
  else
    bn_bwd_reduce_kernel<T, V, RELU, false, false><<<rgrid, l.threads, smem, stream>>>(g, x, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  dim3 block;
  const dim3 grid = elementwise_grid(M, C, V, &block);
  const float nf = (float)(1.0 / (double)M);
  bn_bwd_elemt_kernel<T, V, RELU><<<grid, block, 0, stream>>>(g, x, (T*)p.gx, p.mean, p.invstd, p.weight, p.bias,
                                                              p.sum_dy, p.sum_dy_xmu, nf, M, C);
  return cudaGetLastError();
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

template <typename T>
cudaError_t dispatch_vec(const BnForwardArgs& p, cudaStream_t stream) {
  constexpr int V = DT<T>::kVec;
  const bool vec = p.C % V == 0 && aligned16(p.x) && aligned16(p.y);
  return vec ? forward_t<T, V>(p, stream) : forward_t<T, 1>(p, stream);
}

template <typename T>
cudaError_t dispatch_vec(const BnBackwardArgs& p, cudaStream_t stream) {
  constexpr int V = DT<T>::kVec;
  const bool vec = p.C % V == 0 && aligned16(p.g) && aligned16(p.x) && aligned16(p.gx);
  if (p.relu) return vec ? backward_t<T, V, true>(p, stream) : backward_t<T, 1, true>(p, stream);
  return vec ? backward_t<T, V, false>(p, stream) : backward_t<T, 1, false>(p, stream);
}

}  // namespace

int batchnorm_cl_grid_y(int M, int C) { return aten_grid(M, C).gy; }

template <typename Args>
cudaError_t dispatch_dtype(const Args& p, cudaStream_t stream) {
  if ((int64_t)p.M * p.C == 0) return cudaSuccess;
  switch (p.dtype) {
    case kF32: return dispatch_vec<float>(p, stream);
    case kF16: return dispatch_vec<__half>(p, stream);
    case kBF16: return dispatch_vec<__nv_bfloat16>(p, stream);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_batchnorm_cl_forward(const BnForwardArgs& p, cudaStream_t stream) {
  return dispatch_dtype(p, stream);
}

cudaError_t launch_batchnorm_cl_backward(const BnBackwardArgs& p, cudaStream_t stream) {
  return dispatch_dtype(p, stream);
}

}  // namespace cgx

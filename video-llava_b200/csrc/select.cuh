// Row-selection building blocks shared by the sampler (sampling.cu) and beam search (beam.cu): order-preserving keys
// of fp32 values, the radix select of the k-th largest key, the kept-weight sums of the log-softmax and the
// collection of the n largest keys. One CTA of SEL_THREADS threads per row; the row's keys are staged in shared
// memory.
#pragma once

#include <math.h>

#include "common.cuh"

namespace vcl {

constexpr int SEL_THREADS = 512;
constexpr int SEL_WARPS = SEL_THREADS / 32;

// order-preserving key of any fp32 value; NaN maps to 0, below every number, and -0 to the key of +0, since the two
// compare equal (an arg-max then takes the lower index, as argmax_kernel does)
__device__ __forceinline__ uint32_t order_key32(float x) {
  if (x != x) return 0u;
  const uint32_t b = x == 0.f ? 0u : __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value32(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
constexpr uint32_t KEY32_NEG_INF = 0x007fffffu;   // order_key32(-inf)

// The need-th largest key of skey[0 .. V) (1 <= need <= V): PASSES 8-bit histogram passes from the high byte
// down, each inside the bytes chosen so far. *left receives the rank left inside that key: the key's ties to take,
// counting from the lowest index, after the keys above it.
template <int PASSES, class Key>
__device__ __forceinline__ uint32_t radix_select(const Key* skey, int V, uint32_t need, uint32_t* s_hist,
                                                 uint32_t* s_wcnt, uint32_t* s_sel, uint32_t* left) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t prefix = 0;   // the bytes found so far
  for (int pass = 0; pass < PASSES; ++pass) {
    const int shift = 8 * (PASSES - 1 - pass);
    if (tid < 256) s_hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < V; i += SEL_THREADS) {
      const uint32_t key = skey[i];
      if (pass == 0) atomicAdd(&s_hist[key >> shift], 1u);
      else if ((key >> (shift + 8)) == prefix) atomicAdd(&s_hist[(key >> shift) & 0xffu], 1u);
    }
    __syncthreads();
    // threads 0..255 take the bins from the top down; an inclusive scan of the counts finds the bin in which
    // the count from the top reaches `need`
    uint32_t h = 0, incl = 0;
    if (tid < 256) {
      h = s_hist[255 - tid];
      incl = h;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
      }
      if (lane == 31) s_wcnt[warp] = incl;
    }
    __syncthreads();
    if (tid < 256) {
      for (int w = 0; w < warp; ++w) incl += s_wcnt[w];
      if (incl >= need && incl - h < need) {
        s_sel[0] = 255 - tid;           // the bin
        s_sel[1] = need - (incl - h);   // the rank left inside it
      }
    }
    __syncthreads();
    prefix = pass == 0 ? s_sel[0] : ((prefix << 8) | s_sel[0]);
    need = s_sel[1];
    __syncthreads();                    // s_sel and s_hist are rewritten by the next pass
  }
  *left = need;
  return prefix;
}

// The kept weights w_i = exp(z_i - zmax) of a row (z_i = zval(skey[i]) >= zthr), in one fixed order: every thread
// sums its contiguous run [i_beg, i_end) of the row in index order (*s), then a block scan over the runs gives *excl,
// the sum of the runs before this one, and *W, the row's sum. *last: the run's last index with a nonzero weight.
// The log-softmax of the greedy log-prob rule is lp_j = (z_j - zmax) - logf(W) (DESIGN.md section 3), so every
// caller of this function computes it bit for bit alike. s_sum: SEL_WARPS floats of shared memory.
template <class Key, class ZVal>
__device__ __forceinline__ void kept_weights(const Key* skey, int i_beg, int i_end, ZVal zval, float zthr, float zmax,
                                             float* s_sum, float* s, float* excl, float* W, int* last) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float sum = 0.f;
  int lst = -1;
  for (int i = i_beg; i < i_end; ++i) {
    const float z = zval(skey[i]);
    if (z >= zthr) {
      const float w = expf(z - zmax);
      sum += w;
      if (w > 0.f) lst = i;
    }
  }
  float incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  if (lane == 31) s_sum[warp] = incl;
  __syncthreads();
  float ex = incl - sum, tot = 0.f;
#pragma unroll
  for (int w = 0; w < SEL_WARPS; ++w) {
    if (w < warp) ex += s_sum[w];
    tot += s_sum[w];
  }
  *s = sum; *excl = ex; *W = tot; *last = lst;
}

// The n largest keys of skey[0 .. V) (1 <= n <= V), ties from the lowest index: every key above the n-th largest,
// then its ties (each run's first tie rank from a block scan of the per-run tie counts; the runs are in index
// order). They land in s_top_key / s_top_idx [n] in no particular order. s_cnt: SEL_WARPS words.
template <int PASSES, class Key>
__device__ __forceinline__ void collect_top(const Key* skey, int V, int n, int i_beg, int i_end, uint32_t* s_hist,
                                            uint32_t* s_wcnt, uint32_t* s_sel, uint32_t* s_cnt, int* s_ntop,
                                            uint32_t* s_top_key, int* s_top_idx) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t take;
  const uint32_t kn = radix_select<PASSES>(skey, V, (uint32_t)n, s_hist, s_wcnt, s_sel, &take);
  uint32_t eq = 0;
  for (int i = i_beg; i < i_end; ++i) eq += skey[i] == kn;
  uint32_t eincl = eq;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t m = __shfl_up_sync(0xffffffffu, eincl, o);
    if (lane >= o) eincl += m;
  }
  if (lane == 31) s_cnt[warp] = eincl;
  if (tid == 0) *s_ntop = 0;
  __syncthreads();
  uint32_t rank = eincl - eq;
  for (int w = 0; w < warp; ++w) rank += s_cnt[w];
  for (int i = i_beg; i < i_end; ++i) {
    const uint32_t key = skey[i];
    bool sel = key > kn;
    if (key == kn) sel = rank++ < take;
    if (sel) {
      const int q = atomicAdd(s_ntop, 1);
      s_top_key[q] = key;
      s_top_idx[q] = i;
    }
  }
  __syncthreads();
}

}  // namespace vcl

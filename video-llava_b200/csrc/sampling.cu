// Temperature / top-k sampling of the next token on the device, one CTA per row.
//
// Reference: video_chatgpt/inference.py:105-107 calls generate(do_sample=True, temperature=0.2), i.e.
// transformers' _sample with TemperatureLogitsWarper then TopKLogitsWarper (top_k 50) on fp32 logits. The rules
// (DESIGN.md section 3):
//   x      the row's logits, bf16-rounded values in fp32 storage (GEMV_LOGITS)
//   z_i    fp32(x_i / T), a true division (not a multiply by 1/T)
//   kept   z_i >= z of the k-th largest logit (ties at the threshold are kept, HF's `scores < kth` rule);
//          top_k = 0 or top_k >= V keeps every token; a NaN logit is never kept
//   w_i    exp(z_i - z_max) over the kept tokens, in fp32
//   token  the smallest j whose inclusive prefix sum of w exceeds u * W (W = sum of w); if rounding leaves u * W
//          past the last prefix sum, the last token with a nonzero weight (a -inf logit or an exp that underflows
//          to 0 is never drawn)
//   u      (word0 >> 8) * 2^-24, word0 the first word of Philox4x32-10 with key = the row's 64-bit seed (lo, hi)
//          and counter = (p, 0, 0, 0), p the RoPE position the sampled token takes (cache column - n_pad)
// A row with T = 0, or whose scaled maximum z_max is not finite, takes the arg-max instead: the token
// argmax_kernel gives (lowest index of the largest non-NaN logit, 0 when no logit is above -inf).
//
// The row (4 V bytes) is read once. Because its values are bf16, it is staged in shared memory as 16-bit keys
// whose unsigned order is the order of the values, so the exact k-th largest logit comes from a radix select of
// two 8-bit histogram passes (no sort, any k). Every thread owns a contiguous run of the row; the run sums and a
// block-wide scan over them give the prefix sums in one fixed order, so the token is the same from run to run.
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

constexpr int SM_THREADS = 512;
constexpr int SM_WARPS = SM_THREADS / 32;
constexpr int SM_MAX_V = 80 * 1024;   // the staged row of 16-bit keys: 160 KB of shared memory

__device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) { return __umulhi(a, b); }

// order-preserving key of a bf16 value (the upper half of its fp32 bits); NaN maps to 0, below every number, and
// -0 to the key of +0, since the two compare equal (the arg-max then takes the lower index, as argmax_kernel does)
__device__ __forceinline__ uint32_t order_key(float x) {
  if (x != x) return 0u;
  const uint32_t b = x == 0.f ? 0u : __float_as_uint(x) >> 16;
  return (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  const uint32_t b = (k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu);
  return __uint_as_float(b << 16);
}
constexpr uint32_t KEY_NEG_INF = 0x007fu;   // order_key(-inf)

__global__ void __launch_bounds__(SM_THREADS)
sample_kernel(SampleArgs a) {
  extern __shared__ __align__(16) uint16_t skey[];
  __shared__ unsigned long long s_red[SM_WARPS];
  __shared__ float s_sum[SM_WARPS];
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_wcnt[8];
  __shared__ uint32_t s_sel[2];
  __shared__ int s_pick[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r = blockIdx.x;
  const int V = a.V;
  const int t = a.entry0 + (a.rowmap != nullptr ? a.rowmap[r] : r);
  const float* x = a.logits + (long long)r * a.ld;

  // stage the keys; the largest key with its lowest index (the arg-max, packed so that a max-reduce finds it)
  unsigned long long best = 0;
  constexpr int U = 8;
  for (int i0 = tid; i0 < V; i0 += SM_THREADS * U) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * SM_THREADS;
      v[u] = i < V ? x[i] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * SM_THREADS;
      if (i < V) {
        const uint32_t k = order_key(v[u]);
        skey[i] = (uint16_t)k;
        const unsigned long long p = ((unsigned long long)k << 32) | (0xffffffffu - (uint32_t)i);
        best = p > best ? p : best;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long q = __shfl_xor_sync(0xffffffffu, best, o);
    best = q > best ? q : best;
  }
  if (lane == 0) s_red[warp] = best;
  __syncthreads();
  best = s_red[0];
#pragma unroll
  for (int w = 1; w < SM_WARPS; ++w) best = s_red[w] > best ? s_red[w] : best;
  const uint32_t kmax = (uint32_t)(best >> 32);
  const int amax = kmax > KEY_NEG_INF ? (int)(0xffffffffu - (uint32_t)best) : 0;

  const float T = a.temperature[t];
  const float zmax = __fdiv_rn(key_value(kmax), T);
  if (!(T > 0.f) || !isfinite(zmax)) {   // greedy entry, or no finite scaled maximum: the arg-max
    if (tid == 0) a.out[(long long)r * a.out_stride] = amax;
    return;
  }

  // the k-th largest key: two 8-bit histogram passes (high byte, then low byte inside the chosen high byte)
  const int k = a.top_k[t];
  float zthr = -INFINITY;
  if (k > 0 && k < V) {
    uint32_t need = (uint32_t)k, prefix = 0;   // rank still to find, high byte found by pass 0
    for (int pass = 0; pass < 2; ++pass) {
      if (tid < 256) s_hist[tid] = 0;
      __syncthreads();
      for (int i = tid; i < V; i += SM_THREADS) {
        const uint32_t key = skey[i];
        if (pass == 0) atomicAdd(&s_hist[key >> 8], 1u);
        else if ((key >> 8) == prefix) atomicAdd(&s_hist[key & 0xffu], 1u);
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
    // a NaN at the threshold (k past the numbers of the row) keeps every number
    if (prefix >= KEY_NEG_INF) zthr = __fdiv_rn(key_value(prefix), T);
  }

  // each thread's contiguous run: the sum of its kept weights in index order, then a scan over the runs.
  // Prefix sum of index j (in run t): P_j = excl_t + (the run's own running sum up to j)
  const int run = (V + SM_THREADS - 1) / SM_THREADS;
  const int i_beg = tid * run, i_end = min(i_beg + run, V);
  float s = 0.f;
  int last = -1;                   // the run's last index with a nonzero weight
  for (int i = i_beg; i < i_end; ++i) {
    const float z = __fdiv_rn(key_value(skey[i]), T);
    if (z >= zthr) {
      const float w = expf(z - zmax);
      s += w;
      if (w > 0.f) last = i;
    }
  }
  float incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  if (lane == 31) s_sum[warp] = incl;
  if (tid == 0) { s_pick[0] = 0x7fffffff; s_pick[1] = -1; }
  __syncthreads();
  float excl = incl - s, W = 0.f;
#pragma unroll
  for (int w = 0; w < SM_WARPS; ++w) {
    if (w < warp) excl += s_sum[w];
    W += s_sum[w];
  }

  // Philox4x32-10, key = seed, counter = (p, 0, 0, 0)
  const unsigned long long seed = a.seed[t];
  const int p = a.col + (a.col_dev != nullptr ? a.col_dev[r] : 0) - (a.n_pad != nullptr ? a.n_pad[t] : 0);
  uint32_t c0 = (uint32_t)p, c1 = 0, c2 = 0, c3 = 0;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int round = 0; round < 10; ++round) {
    const uint32_t hi0 = mulhi32(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = mulhi32(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  const float uW = (float)(c0 >> 8) * 5.9604644775390625e-8f * W;   // u = (word0 >> 8) * 2^-24

  // the first index whose inclusive prefix sum exceeds u * W (P_j grows with j inside a run, so a run whose
  // last prefix sum does not exceed u * W holds none)
  if (excl + s > uW) {
    float acc = 0.f;
    for (int i = i_beg; i < i_end; ++i) {
      const float z = __fdiv_rn(key_value(skey[i]), T);
      if (z >= zthr) {
        const float w = expf(z - zmax);
        acc += w;
        if (w > 0.f && excl + acc > uW) {   // (a zero weight never starts an interval)
          atomicMin(&s_pick[0], i);
          break;
        }
      }
    }
  }
  if (last >= 0) atomicMax(&s_pick[1], last);
  __syncthreads();
  if (tid == 0) a.out[(long long)r * a.out_stride] = s_pick[0] != 0x7fffffff ? s_pick[0] : s_pick[1];
}

}  // namespace

int launch_sample(const SampleArgs& a, cudaStream_t stream) {
  VCL_REQUIRE(a.B >= 0 && a.V > 0 && a.V <= SM_MAX_V && a.ld >= a.V,
              "sample: V=%d outside 1..%d or row pitch %lld < V", a.V, SM_MAX_V, a.ld);
  VCL_REQUIRE(a.logits && a.temperature && a.top_k && a.seed && a.out, "sample: null argument");
  if (a.B == 0) return 0;
  static bool attr = false;
  if (!attr) {
    VCL_CUDA_OK(cudaFuncSetAttribute(sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_MAX_V * 2));
    attr = true;
  }
  const size_t smem = ((size_t)a.V * 2 + 15) / 16 * 16;
  sample_kernel<<<a.B, SM_THREADS, smem, stream>>>(a);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

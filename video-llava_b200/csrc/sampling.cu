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
// Log-probabilities (an entry with top_n >= 0; DESIGN.md section 3): s = z over the kept tokens (a greedy row: s = x,
// every non-NaN token kept, as if T = 1 and k = 0), m = z_max, W the sum of w above in its fixed order, and
// lp(j) = (s_j - m) - logf(W) for the chosen token and the top_n kept tokens of largest s (ties: lowest index),
// selected by the same radix select and sorted by one warp. A row without a finite maximum reports NaN.
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

// The need-th largest key of skey[0 .. V) (1 <= need <= V): two 8-bit histogram passes (high byte, then low byte
// inside the chosen high byte). *left receives the rank left inside that key: the key's ties to take, counting
// from the lowest index, after the keys above it.
__device__ __forceinline__ uint32_t radix_select(const uint16_t* skey, int V, uint32_t need, uint32_t* s_hist,
                                                 uint32_t* s_wcnt, uint32_t* s_sel, uint32_t* left) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t prefix = 0;   // high byte found by pass 0
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
  *left = need;
  return prefix;
}

// place q of a log-prob row
__device__ __forceinline__ void put_lp(const SampleArgs& a, long long row, int q, int id, float lp) {
  const long long o = row + q;
  a.lp_id[o] = id;
  a.lp_val[o] = lp;
}

// (min 1 block: the staged row fills shared memory anyway; without it ptxas holds 40 registers and spills)
__global__ void __launch_bounds__(SM_THREADS, 1)
sample_kernel(SampleArgs a) {
  extern __shared__ __align__(16) uint16_t skey[];
  __shared__ unsigned long long s_red[SM_WARPS];
  __shared__ float s_sum[SM_WARPS];
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_wcnt[8];
  __shared__ uint32_t s_sel[2];
  __shared__ int s_pick[2];
  __shared__ uint32_t s_cnt[SM_WARPS];
  __shared__ uint32_t s_top_key[VCL_LOGPROBS_MAX];
  __shared__ int s_top_idx[VCL_LOGPROBS_MAX];
  __shared__ int s_ntop;
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

  // log-probs: the chosen token and n_lp alternatives (off: -1); a greedy row then scores s = x (T = 1, k = 0)
  const int n_lp = a.top_n != nullptr ? a.top_n[t] : -1;
  const float T0 = a.temperature[t];
  const bool greedy = !(T0 > 0.f);
  const float T = greedy ? 1.f : T0;
  auto position = [&]() {
    return a.col + (a.col_dev != nullptr ? a.col_dev[r] : 0) - (a.n_pad != nullptr ? a.n_pad[t] : 0);
  };
  const float zmax = __fdiv_rn(key_value(kmax), T);
  if ((greedy && n_lp < 0) || !isfinite(zmax)) {   // greedy entry, or no finite scaled maximum: the arg-max
    if (tid == 0) a.out[(long long)r * a.out_stride] = amax;
    if (n_lp >= 0) {
      const int p = position();
      if (p >= 0 && p < a.lp_rows && tid <= n_lp) {
        const long long row = (long long)t * a.lp_entry + (long long)p * a.lp_pos;
        put_lp(a, row, tid, tid == 0 ? amax : -1, __int_as_float(0x7fffffff));
      }
    }
    return;
  }

  // the k-th largest key: the radix select
  const int k = greedy ? 0 : a.top_k[t];
  float zthr = -INFINITY;
  if (k > 0 && k < V) {
    uint32_t left;
    const uint32_t prefix = radix_select(skey, V, (uint32_t)k, s_hist, s_wcnt, s_sel, &left);
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

  int tok = amax;
  if (!greedy) {
    // Philox4x32-10, key = seed, counter = (p, 0, 0, 0)
    const unsigned long long seed = a.seed[t];
    const int p = position();
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
    tok = s_pick[0] != 0x7fffffff ? s_pick[0] : s_pick[1];
  }
  if (tid == 0) a.out[(long long)r * a.out_stride] = tok;
  if (n_lp < 0) return;

  // log-probs of the token at position p: lp(j) = (s_j - m) - log W
  const int p = position();
  if (p < 0 || p >= a.lp_rows) return;
  const long long row = (long long)t * a.lp_entry + (long long)p * a.lp_pos;
  const float lw = logf(W);
  if (tid == 0) put_lp(a, row, 0, tok, (__fdiv_rn(key_value(skey[tok]), T) - zmax) - lw);
  if (n_lp == 0) return;
  const int n_sel = min(n_lp, V);
  // the n_sel largest keys: every key above the n_sel-th largest, then its ties from the lowest index (each run's
  // first tie rank from a block scan of the per-run tie counts; the runs are in index order)
  uint32_t take;
  const uint32_t kn = radix_select(skey, V, (uint32_t)n_sel, s_hist, s_wcnt, s_sel, &take);
  uint32_t eq = 0;
  for (int i = i_beg; i < i_end; ++i) eq += skey[i] == kn;
  uint32_t eincl = eq;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(0xffffffffu, eincl, o);
    if (lane >= o) eincl += n;
  }
  if (lane == 31) s_cnt[warp] = eincl;
  if (tid == 0) s_ntop = 0;
  __syncthreads();
  uint32_t rank = eincl - eq;
  for (int w = 0; w < warp; ++w) rank += s_cnt[w];
  for (int i = i_beg; i < i_end; ++i) {
    const uint32_t key = skey[i];
    bool sel = key > kn;
    if (key == kn) sel = rank++ < take;
    if (sel) {
      const int q = atomicAdd(&s_ntop, 1);
      s_top_key[q] = key;
      s_top_idx[q] = i;
    }
  }
  __syncthreads();
  // one warp sorts them: key descending, then index ascending. A token the top-k rule drops (or a NaN) is reported
  // as -1 / -inf; those sort after every kept token, since a larger key never has a smaller s
  if (warp == 0 && lane < n_lp) {
    int id = -1;
    float lp = -INFINITY;
    int place = lane;
    if (lane < n_sel) {
      const uint32_t key = s_top_key[lane];
      const int idx = s_top_idx[lane];
      place = 0;
      for (int j = 0; j < n_sel; ++j) {
        const uint32_t kj = s_top_key[j];
        place += kj > key || (kj == key && s_top_idx[j] < idx);
      }
      const float z = __fdiv_rn(key_value(key), T);
      if (z >= zthr) { id = idx; lp = (z - zmax) - lw; }
    }
    put_lp(a, row, 1 + place, id, lp);
  }
}

}  // namespace

int launch_sample(const SampleArgs& a, cudaStream_t stream) {
  VCL_REQUIRE(a.B >= 0 && a.V > 0 && a.V <= SM_MAX_V && a.ld >= a.V,
              "sample: V=%d outside 1..%d or row pitch %lld < V", a.V, SM_MAX_V, a.ld);
  VCL_REQUIRE(a.logits && a.temperature && a.top_k && a.seed && a.out, "sample: null argument");
  VCL_REQUIRE(a.top_n == nullptr || (a.lp_id && a.lp_val), "sample: log-probs need their outputs");
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

// Temperature / top-k / top-p sampling of the next token on the device, with HF's repetition penalty, one CTA per
// row.
//
// Reference: video_chatgpt/inference.py:105-107 calls generate(do_sample=True, temperature=0.2), i.e.
// transformers' _sample with TemperatureLogitsWarper then TopKLogitsWarper (top_k 50) on fp32 logits; HF runs
// RepetitionPenaltyLogitsProcessor before them and TopPLogitsWarper after them. The rules (DESIGN.md section 3):
//   x      the row's logits, bf16-rounded values in fp32 storage (GEMV_LOGITS)
//   x'     the penalized logit (repetition penalty r != 1 only): for a token of the entry's token set,
//          x < 0 ? fp32(x * r) : fp32(x / r); every other token keeps x
//   z_i    fp32(x'_i / T), a true division (not a multiply by 1/T)
//   kept   z_i >= z of the k-th largest logit (ties at the threshold are kept, HF's `scores < kth` rule);
//          top_k = 0 or top_k >= V keeps every token; a NaN logit is never kept
//   top-p  (p < 1, sampled rows) of the kept tokens, those whose key is the largest, or whose mass strictly above
//          it M is below p * W, in the fixed-point rule at top_p_threshold
//   w_i    exp(z_i - z_max) over the kept tokens, in fp32
//   token  the smallest j whose inclusive prefix sum of w exceeds u * W (W = sum of w); if rounding leaves u * W
//          past the last prefix sum, the last token with a nonzero weight (a -inf logit or an exp that underflows
//          to 0 is never drawn)
//   u      (word0 >> 8) * 2^-24, word0 the first word of Philox4x32-10 with key = the row's 64-bit seed (lo, hi)
//          and counter = (p, 0, 0, 0), p the RoPE position the sampled token takes (cache column - n_pad)
// A row with T = 0, or whose scaled maximum z_max is not finite, takes the arg-max instead: the token
// argmax_kernel gives (lowest index of the largest non-NaN logit -- of x' on the 32-bit path -- 0 when no logit
// is above -inf).
//
// Log-probabilities (an entry with top_n >= 0; DESIGN.md section 3): s = z over the kept tokens (a greedy row: s = x',
// every non-NaN token kept, as if T = 1 and k = 0), m = z_max, W the sum of w above in its fixed order, and
// lp(j) = (s_j - m) - logf(W) for the chosen token and the top_n kept tokens of largest s (ties: lowest index),
// selected by the same radix select and sorted by one warp. A row without a finite maximum reports NaN.
//
// The row (4 V bytes) is read once and staged in shared memory as keys whose unsigned order is the order of the
// values, so the exact k-th largest logit comes from a radix select of 8-bit histogram passes (no sort, any k).
// Every thread owns a contiguous run of the row; the run sums and a block-wide scan over them give the prefix sums
// in one fixed order, so the token is the same from run to run. Two instances:
//   16-bit keys (the launch has no top_p / repetition table): the values are bf16, so the key of x is its upper
//          half; T is applied when a key is read back. Two select passes; V <= SM_MAX_V.
//   32-bit keys (SampleArgs::top_p set): the key of z itself, since a penalized z is not a bf16 value. Four select
//          passes, then the top-p threshold; V <= VCL_SAMPLE_WIDE_MAX_V. For r = 1 and p = 1 its tokens and
//          log-probs are the 16-bit instance's bit for bit (z of a larger x is never smaller, so the k-th largest z
//          is fp32(k-th largest x / T)). The sampler adds the token it picks to the entry's token set.
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

constexpr int SM_THREADS = 512;
constexpr int SM_WARPS = SM_THREADS / 32;
constexpr int SM_MAX_V = 80 * 1024;   // the staged row of 16-bit keys: 160 KB of shared memory
constexpr int SM_MAX_V_WIDE = VCL_SAMPLE_WIDE_MAX_V;   // 32-bit keys: 224 KB, of the 227 KB a block may take

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

// the same over all 32 bits of any fp32 value
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
    for (int i = tid; i < V; i += SM_THREADS) {
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

// fixed-point mass of a kept token: q = rint(w * 2^36), w = exp(z - z_max) in fp32 (so q <= 2^36 and the masses of
// a row of up to 2^17 tokens sum exactly, below 2^53, in any order)
__device__ __forceinline__ unsigned long long fixed_mass(float w) { return __float2ull_rn(w * 68719476736.f); }

// The top-p threshold of a sampled row on the 32-bit keys: with q the fixed-point masses of the kept tokens
// (z >= zthr), Q their sum and F(k) the sum of q over the kept keys strictly above k, the smallest key tau such
// that every kept key k >= tau has F(k) < p * Q (fp64 product of fp64(p) and Q; tau = the largest key when that is
// 0). Keys >= tau are then exactly the kept keys with F(k) < p * Q, ties whole. Four 8-bit passes from the high
// byte, each histogramming the masses inside the bytes chosen so far; in a pass the chosen bin is the lowest one
// whose mass above (those of the higher bins, plus the mass above the prefix) is below p * Q. Integer sums: the
// same bits on every run. s_mass: 256 + SM_WARPS 64-bit words.
__device__ __forceinline__ uint32_t top_p_threshold(const uint32_t* skey, int V, float zthr, float zmax, float p,
                                                    uint32_t kmax, unsigned long long* s_mass, uint32_t* s_sel) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned long long* s_wm = s_mass + 256;
  __shared__ unsigned long long s_base;
  uint32_t prefix = 0;
  unsigned long long base = 0;   // the mass above the prefix
  double P = 0.0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 8 * (3 - pass);
    if (tid < 256) s_mass[tid] = 0;
    __syncthreads();
    // most keys share their high bytes, so the lanes of a warp that hit one bin add their masses first (exactly:
    // q <= 2^36 is summed as two 18-bit halves) and one of them does the shared-memory atomic
    for (int i0 = 0; i0 < V; i0 += SM_THREADS) {
      const int i = i0 + tid;
      uint32_t bin = 256;             // none
      unsigned long long q = 0;
      if (i < V) {
        const uint32_t key = skey[i];
        const float z = key_value32(key);
        if ((pass == 0 || (key >> (shift + 8)) == prefix) && z >= zthr) {
          q = fixed_mass(expf(z - zmax));
          if (q != 0) bin = (key >> shift) & 0xffu;
        }
      }
      const uint32_t peers = __match_any_sync(0xffffffffu, bin);
      const uint32_t lo = __reduce_add_sync(peers, (uint32_t)(q & 0x3ffffu));
      const uint32_t hi = __reduce_add_sync(peers, (uint32_t)(q >> 18));
      if (bin < 256 && lane == __ffs(peers) - 1)
        atomicAdd(&s_mass[bin], ((unsigned long long)hi << 18) + lo);
    }
    __syncthreads();
    unsigned long long h = 0, incl = 0;
    if (tid < 256) {
      h = s_mass[255 - tid];
      incl = h;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
      }
      if (lane == 31) s_wm[warp] = incl;
    }
    __syncthreads();
    if (pass == 0) {   // Q = the whole kept mass
      unsigned long long Q = 0;
      for (int w = 0; w < 8; ++w) Q += s_wm[w];
      P = (double)p * (double)Q;
      if (!(P > 0.0)) return kmax;   // (uniform: every thread sees the same Q)
    }
    if (tid < 256) {
      for (int w = 0; w < warp; ++w) incl += s_wm[w];
      const bool below = (double)(base + incl - h) < P;   // the mass above this bin
      const bool next = tid < 255 && (double)(base + incl) < P;   // ... and above the next lower bin
      if (below && !next) {
        s_sel[0] = 255 - tid;
        s_base = base + incl - h;
      }
    }
    __syncthreads();
    prefix = (prefix << 8) | s_sel[0];
    base = s_base;
    __syncthreads();
  }
  return prefix;
}

// place q of a log-prob row
__device__ __forceinline__ void put_lp(const SampleArgs& a, long long row, int q, int id, float lp) {
  const long long o = row + q;
  a.lp_id[o] = id;
  a.lp_val[o] = lp;
}

// (min 1 block: the staged row fills shared memory anyway; without it ptxas holds 40 registers and spills)
template <bool WIDE>
__global__ void __launch_bounds__(SM_THREADS, 1)
sample_kernel(SampleArgs a) {
  using Key = typename std::conditional<WIDE, uint32_t, uint16_t>::type;
  extern __shared__ __align__(16) unsigned char s_stage[];
  Key* skey = reinterpret_cast<Key*>(s_stage);
  __shared__ unsigned long long s_red[SM_WARPS];
  __shared__ float s_sum[SM_WARPS];
  // the count histogram; on the 32-bit path also the 64-bit masses of top_p_threshold (256 + SM_WARPS words)
  __shared__ __align__(8) uint32_t s_hist[WIDE ? 2 * (256 + SM_WARPS) : 256];
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

  // the 32-bit path stages z: the temperature (greedy: 1), the penalty (1: off) and the entry's token set, a bitmap
  // of tset_words words
  float T_stage = 1.f, rep = 1.f;
  const uint32_t* tset = nullptr;
  if constexpr (WIDE) {
    const float T0 = a.temperature[t];
    T_stage = T0 > 0.f ? T0 : 1.f;
    rep = a.rep[t];
    if (a.tset != nullptr) tset = a.tset + (long long)t * a.tset_words;
  }

  // stage the keys; the largest key with its lowest index (the arg-max, packed so that a max-reduce finds it). The
  // 32-bit path also finds the arg-max of x' itself: z = x' / T can tie (or overflow) where x' does not, and the
  // arg-max fallback must not depend on which path a call takes
  unsigned long long best = 0, best_x = 0;
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
        uint32_t k;
        if constexpr (WIDE) {
          float xp = v[u];
          if (rep != 1.f && tset != nullptr && ((__ldg(tset + (i >> 5)) >> (i & 31)) & 1u))
            xp = xp < 0.f ? __fmul_rn(xp, rep) : __fdiv_rn(xp, rep);
          k = order_key32(__fdiv_rn(xp, T_stage));
          const unsigned long long px = ((unsigned long long)order_key32(xp) << 32) | (0xffffffffu - (uint32_t)i);
          best_x = px > best_x ? px : best_x;
        } else {
          k = order_key(v[u]);
        }
        skey[i] = (Key)k;
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
  int amax = kmax > (WIDE ? KEY32_NEG_INF : KEY_NEG_INF) ? (int)(0xffffffffu - (uint32_t)best) : 0;
  if constexpr (WIDE) {
    __shared__ unsigned long long s_red_x[SM_WARPS];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long q = __shfl_xor_sync(0xffffffffu, best_x, o);
      best_x = q > best_x ? q : best_x;
    }
    if (lane == 0) s_red_x[warp] = best_x;
    __syncthreads();
    best_x = s_red_x[0];
#pragma unroll
    for (int w = 1; w < SM_WARPS; ++w) best_x = s_red_x[w] > best_x ? s_red_x[w] : best_x;
    amax = (uint32_t)(best_x >> 32) > KEY32_NEG_INF ? (int)(0xffffffffu - (uint32_t)best_x) : 0;
  }

  // the token: to the output, and on the 32-bit path into the entry's token set (one row per entry and launch)
  auto emit = [&](int tok) {
    a.out[(long long)r * a.out_stride] = tok;
    if constexpr (WIDE) {
      if (a.tset != nullptr) atomicOr(a.tset + (long long)t * a.tset_words + (tok >> 5), 1u << (tok & 31));
    }
  };

  // log-probs: the chosen token and n_lp alternatives (off: -1); a greedy row then scores s = x' (T = 1, k = 0)
  const int n_lp = a.top_n != nullptr ? a.top_n[t] : -1;
  const float T0 = a.temperature[t];
  const bool greedy = !(T0 > 0.f);
  const float T = greedy ? 1.f : T0;
  // z of a staged key
  auto zval = [&](uint32_t key) -> float {
    if constexpr (WIDE) return key_value32(key);
    else return __fdiv_rn(key_value(key), T);
  };
  auto position = [&]() {
    return a.col + (a.col_dev != nullptr ? a.col_dev[r] : 0) - (a.n_pad != nullptr ? a.n_pad[t] : 0);
  };
  const float zmax = zval(kmax);
  if ((greedy && n_lp < 0) || !isfinite(zmax)) {   // greedy entry, or no finite scaled maximum: the arg-max
    if (tid == 0) emit(amax);
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
    const uint32_t prefix = radix_select<WIDE ? 4 : 2>(skey, V, (uint32_t)k, s_hist, s_wcnt, s_sel, &left);
    // a NaN at the threshold (k past the numbers of the row) keeps every number
    if (prefix >= (WIDE ? KEY32_NEG_INF : KEY_NEG_INF)) zthr = zval(prefix);
  }
  if constexpr (WIDE) {   // top-p narrows the kept set to the keys >= tau
    const float top_p = a.top_p[t];
    if (!greedy && top_p < 1.f) {
      const uint32_t tau = top_p_threshold(reinterpret_cast<const uint32_t*>(skey), V, zthr, zmax, top_p, kmax,
                                           reinterpret_cast<unsigned long long*>(s_hist), s_sel);
      const float ztau = key_value32(tau);
      if (ztau > zthr) zthr = ztau;
      __syncthreads();   // s_hist / s_sel are reused below
    }
  }

  // each thread's contiguous run: the sum of its kept weights in index order, then a scan over the runs.
  // Prefix sum of index j (in run t): P_j = excl_t + (the run's own running sum up to j)
  const int run = (V + SM_THREADS - 1) / SM_THREADS;
  const int i_beg = tid * run, i_end = min(i_beg + run, V);
  float s = 0.f;
  int last = -1;                   // the run's last index with a nonzero weight
  for (int i = i_beg; i < i_end; ++i) {
    const float z = zval(skey[i]);
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
        const float z = zval(skey[i]);
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
  if (tid == 0) emit(tok);
  if (n_lp < 0) return;

  // log-probs of the token at position p: lp(j) = (s_j - m) - log W
  const int p = position();
  if (p < 0 || p >= a.lp_rows) return;
  const long long row = (long long)t * a.lp_entry + (long long)p * a.lp_pos;
  const float lw = logf(W);
  if (tid == 0) put_lp(a, row, 0, tok, (zval(skey[tok]) - zmax) - lw);
  if (n_lp == 0) return;
  const int n_sel = min(n_lp, V);
  // the n_sel largest keys: every key above the n_sel-th largest, then its ties from the lowest index (each run's
  // first tie rank from a block scan of the per-run tie counts; the runs are in index order)
  uint32_t take;
  const uint32_t kn = radix_select<WIDE ? 4 : 2>(skey, V, (uint32_t)n_sel, s_hist, s_wcnt, s_sel, &take);
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
  // one warp sorts them: key descending, then index ascending. A token the top-k / top-p rules drop (or a NaN) is
  // reported as -1 / -inf; those sort after every kept token, since a larger key never has a smaller s
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
      const float z = zval(key);
      if (z >= zthr) { id = idx; lp = (z - zmax) - lw; }
    }
    put_lp(a, row, 1 + place, id, lp);
  }
}

// dst[id >> 5] |= 1 << (id & 31) for ids[0 .. n), after the block has cleared dst[0 .. words)
__global__ void token_set_kernel(uint32_t* dst, int words, const long long* ids, int n, int V) {
  for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = 0u;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const long long id = ids[i];
    if (id >= 0 && id < V) atomicOr(dst + (id >> 5), 1u << (id & 31));
  }
}

}  // namespace

int launch_sample(const SampleArgs& a, cudaStream_t stream) {
  const bool wide = a.top_p != nullptr;
  const int max_v = wide ? SM_MAX_V_WIDE : SM_MAX_V;
  VCL_REQUIRE(a.B >= 0 && a.V > 0 && a.V <= max_v && a.ld >= a.V,
              "sample: V=%d outside 1..%d or row pitch %lld < V", a.V, max_v, a.ld);
  VCL_REQUIRE(a.logits && a.temperature && a.top_k && a.seed && a.out, "sample: null argument");
  VCL_REQUIRE(a.top_n == nullptr || (a.lp_id && a.lp_val), "sample: log-probs need their outputs");
  VCL_REQUIRE(!wide || (a.rep && (a.tset == nullptr || a.tset_words >= (a.V + 31) / 32)),
              "sample: the 32-bit path needs the repetition penalties and a token set of %d words", (a.V + 31) / 32);
  if (a.B == 0) return 0;
  if (wide) {
    static bool attr = false;
    if (!attr) {
      VCL_CUDA_OK(cudaFuncSetAttribute(sample_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SM_MAX_V_WIDE * 4));
      attr = true;
    }
    const size_t smem = ((size_t)a.V * 4 + 15) / 16 * 16;
    sample_kernel<true><<<a.B, SM_THREADS, smem, stream>>>(a);
  } else {
    static bool attr = false;
    if (!attr) {
      VCL_CUDA_OK(cudaFuncSetAttribute(sample_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       SM_MAX_V * 2));
      attr = true;
    }
    const size_t smem = ((size_t)a.V * 2 + 15) / 16 * 16;
    sample_kernel<false><<<a.B, SM_THREADS, smem, stream>>>(a);
  }
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_token_set(uint32_t* dst, int words, const long long* ids, int n, int V, cudaStream_t stream) {
  token_set_kernel<<<1, 1024, 0, stream>>>(dst, words, ids, n, V);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

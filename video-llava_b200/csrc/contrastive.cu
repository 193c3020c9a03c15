// Contrastive search on the device (Su et al. 2022; transformers <= 4.55 _contrastive_search / _ranking_fast with
// penalty_alpha = a and top_k = k; DESIGN.md section 3, "Contrastive search"). Per prompt b and step:
//   p_j      exp(lp_j), lp the sampler's greedy log-prob rule on the logits row z of the prompt's last column
//            (select.cuh's kept_weights, so lp is vcl_op_sample_logprobs' value bit for bit)
//   c_1..k   the k largest p, best first, ties to the lower token id (radix select on the keys of p)
//   g_j      the final-RMSNorm row (bf16) of candidate j, decoded as its own cache clip at the same column
//   s_j      max over the prompt's real context rows h of cos(h, g_j) = dot(h, g_j) / (|h| |g_j|), fp32: every dot
//            and squared norm is one warp's sum, lane l taking elements 8c .. 8c+7 of every chunk c = l (mod 32) in
//            ascending order by fmaf, then the xor butterfly 16, 8, 4, 2, 1; |x| = sqrtf of the squared norm, the
//            cosine __fdiv_rn(dot, __fmul_rn(|h|, |g|)); a NaN cosine is skipped by the max
//   score_j  (1 - a) * p_j - a * s_j, each operation rounded once (no contraction); j* the largest, ties to lower j
// The chosen row g_{j*} and its norm are appended to the context, its logits row is the next step's z.
//
// cs_candidates_kernel  one CTA per prompt: p, the top k and the tokens each of the prompt's k clips feeds next
// cs_sim_kernel         CTAs per (row split, candidate group, prompt): one pass over the context rows serves every
//                       candidate of the group; the per-CTA maxima meet in an atomicMax on the cosine's order key
// cs_pick_kernel        one CTA per prompt: scores, pick, step record, the appended context row and its norm
// cs_fork_kernel        the chosen clip's newest cache column copied into the prompt's other clips
// cs_norm_kernel        the fp32 norms of the prefill's context rows (one warp per row, computed once per row)
#include <math.h>

#include "common.cuh"
#include "kernels.h"
#include "select.cuh"

namespace vcl {

namespace {

constexpr int CS_KG = 8;        // candidates per cs_sim_kernel CTA (their rows sit in shared memory)
constexpr int CS_SPLIT = 16;    // row splits per (prompt, candidate group)
constexpr int CS_MAX_D = 8192;

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  f[0] = bf16lo(u.x); f[1] = bf16hi(u.x); f[2] = bf16lo(u.y); f[3] = bf16hi(u.y);
  f[4] = bf16lo(u.z); f[5] = bf16hi(u.z); f[6] = bf16lo(u.w); f[7] = bf16hi(u.w);
}

// the cache clip of candidate j of prompt b (by_clip), or row b * k + j
__device__ __forceinline__ int cs_row(const CsArgs& a, int b, int j) {
  if (!a.by_clip) return b * a.k + j;
  return j == 0 ? b : a.B + b * (a.k - 1) + j - 1;
}

// one warp's dot product of two bf16 rows of D elements (D % 8 == 0) in the order stated above
__device__ __forceinline__ float warp_dot(const bf16* x, const bf16* y, int D) {
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
  for (int c = lane; c < (D >> 3); c += 32) {
    float u[8], v[8];
    unpack8(*reinterpret_cast<const uint4*>(x + c * 8), u);
    unpack8(*reinterpret_cast<const uint4*>(y + c * 8), v);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc = fmaf(u[e], v[e], acc);
  }
  return warp_sum(acc);
}

__global__ void __launch_bounds__(SEL_THREADS, 1) cs_candidates_kernel(CsArgs a) {
  extern __shared__ __align__(16) uint32_t skey[];
  __shared__ uint32_t s_max[SEL_WARPS];
  __shared__ float s_sum[SEL_WARPS];
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_wcnt[8];
  __shared__ uint32_t s_sel[2];
  __shared__ uint32_t s_cnt[SEL_WARPS];
  __shared__ int s_ntop;
  __shared__ uint32_t s_top_key[VCL_CS_MAX_K];
  __shared__ int s_top_idx[VCL_CS_MAX_K];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x, k = a.k, V = a.V;
  const int row = a.first ? b : cs_row(a, b, a.chosen[b]);
  const float* x = a.logits + (long long)row * a.ld;

  uint32_t best = 0;
  for (int i = tid; i < V; i += SEL_THREADS) {
    const uint32_t key = order_key32(x[i]);
    skey[i] = key;
    best = key > best ? key : best;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t q = __shfl_xor_sync(0xffffffffu, best, o);
    best = q > best ? q : best;
  }
  if (lane == 0) s_max[warp] = best;
  __syncthreads();
  best = s_max[0];
#pragma unroll
  for (int w = 1; w < SEL_WARPS; ++w) best = s_max[w] > best ? s_max[w] : best;
  const float m = key_value32(best);

  const int run = (V + SEL_THREADS - 1) / SEL_THREADS;
  const int i_beg = tid * run, i_end = min(i_beg + run, V);
  const bool finite = isfinite(m);   // (uniform)
  float lw = 0.f;
  if (finite) {
    float s, excl, W;
    int last;
    kept_weights(skey, i_beg, i_end, [](uint32_t key) { return key_value32(key); }, -INFINITY, m, s_sum, &s, &excl,
                 &W, &last);
    lw = logf(W);
  }
  // each key becomes the key of p = expf(lp); without a finite maximum every p is NaN (key 0)
  for (int i = i_beg; i < i_end; ++i) {
    const float lp = __fsub_rn(__fsub_rn(key_value32(skey[i]), m), lw);
    skey[i] = finite ? order_key32(expf(lp)) : 0u;
  }
  __syncthreads();
  collect_top<4>(skey, V, k, i_beg, i_end, s_hist, s_wcnt, s_sel, s_cnt, &s_ntop, s_top_key, s_top_idx);
  if (tid < k) {   // place by (p desc, token asc)
    const uint32_t key = s_top_key[tid];
    const int t = s_top_idx[tid];
    int r = 0;
    for (int u = 0; u < k; ++u) r += s_top_key[u] > key || (s_top_key[u] == key && s_top_idx[u] < t);
    a.cand_tok[b * k + r] = t;
    a.cand_p[b * k + r] = key_value32(key);
    a.tok_next[cs_row(a, b, r)] = t;
  }
}

__global__ void __launch_bounds__(256) cs_sim_kernel(CsArgs a) {
  extern __shared__ __align__(16) bf16 sg[];   // [CS_KG][D]
  __shared__ float s_gn[CS_KG];
  const int D = a.D, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.z, j0 = blockIdx.y * CS_KG, kg = min(CS_KG, a.k - j0);
  const int nch = D >> 3;
  for (int e = threadIdx.x; e < kg * nch; e += blockDim.x) {
    const int j = e / nch, c = e - j * nch;
    *reinterpret_cast<uint4*>(sg + (size_t)j * D + c * 8) =
        *reinterpret_cast<const uint4*>(a.hid + (long long)cs_row(a, b, j0 + j) * a.ldh + c * 8);
  }
  __syncthreads();
  if (warp < kg) {
    const float gn = sqrtf(warp_dot(sg + (size_t)warp * D, sg + (size_t)warp * D, D));
    if (lane == 0) {
      s_gn[warp] = gn;
      if (blockIdx.x == 0) a.gnorm[b * a.k + j0 + warp] = gn;
    }
  }
  __syncthreads();
  const int col = a.ctl[3] + a.ctl[0] + a.step;   // this step's column: the context is [n_pad[b], col)
  const bf16* ctx = a.ctx + (long long)b * a.ctx_rows * D;
  float mx[CS_KG];
#pragma unroll
  for (int j = 0; j < CS_KG; ++j) mx[j] = -INFINITY;
  for (int r = a.n_pad[b] + blockIdx.x * 8 + warp; r < col; r += CS_SPLIT * 8) {
    const bf16* hr = ctx + (long long)r * D;
    float acc[CS_KG];
#pragma unroll
    for (int j = 0; j < CS_KG; ++j) acc[j] = 0.f;
    for (int c = lane; c < nch; c += 32) {
      float u[8];
      unpack8(ld_nc_v4(hr + c * 8), u);
#pragma unroll
      for (int j = 0; j < CS_KG; ++j) {
        if (j < kg) {
          float v[8];
          unpack8(*reinterpret_cast<const uint4*>(sg + (size_t)j * D + c * 8), v);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[j] = fmaf(u[e], v[e], acc[j]);
        }
      }
    }
    const float hn = a.ctx_norm[(long long)b * a.ctx_rows + r];
#pragma unroll
    for (int j = 0; j < CS_KG; ++j) {
      const float dot = warp_sum(acc[j]);
      if (j < kg) mx[j] = fmaxf(mx[j], __fdiv_rn(dot, __fmul_rn(hn, s_gn[j])));
    }
  }
  if (lane == 0)
    for (int j = 0; j < kg; ++j) atomicMax(a.sim_key + b * a.k + j0 + j, order_key32(mx[j]));
}

__global__ void __launch_bounds__(128) cs_pick_kernel(CsArgs a) {
  __shared__ float s_score[VCL_CS_MAX_K];
  __shared__ int s_pick;
  const int b = blockIdx.x, k = a.k, tid = threadIdx.x;
  const int t = a.ctl[0] + a.step, col = a.ctl[3] + t;
  float* rec = a.rec + ((long long)a.step * a.B + b) * (2 + 4 * k);
  const float alpha = *a.alpha;
  if (tid < k) {
    unsigned int* sk = a.sim_key + b * k + tid;
    const float s = key_value32(*sk);
    *sk = 0u;   // ready for the next step's atomicMax
    const float p = a.cand_p[b * k + tid];
    const float score = __fsub_rn(__fmul_rn(__fsub_rn(1.f, alpha), p), __fmul_rn(alpha, s));
    s_score[tid] = score;
    rec[2 + tid] = (float)a.cand_tok[b * k + tid];
    rec[2 + k + tid] = p;
    rec[2 + 2 * k + tid] = s;
    rec[2 + 3 * k + tid] = score;
  }
  __syncthreads();
  if (tid == 0) {
    int jb = 0;
    uint32_t kb = order_key32(s_score[0]);
    for (int j = 1; j < k; ++j) {
      const uint32_t kj = order_key32(s_score[j]);
      if (kj > kb) { kb = kj; jb = j; }
    }
    s_pick = jb;
    a.chosen[b] = jb;
    const int tok = a.cand_tok[b * k + jb];
    rec[0] = (float)tok;
    rec[1] = (float)jb;
    if (a.tok_out != nullptr) a.tok_out[(long long)a.step * a.B + b] = tok;
    a.ctx_norm[(long long)b * a.ctx_rows + col] = a.gnorm[b * k + jb];
  }
  __syncthreads();
  const uint4* src = reinterpret_cast<const uint4*>(a.hid + (long long)cs_row(a, b, s_pick) * a.ldh);
  uint4* dst = reinterpret_cast<uint4*>(a.ctx + ((long long)b * a.ctx_rows + col) * a.D);
  for (int c = tid; c < (a.D >> 3); c += blockDim.x) dst[c] = src[c];
}

// one CTA per (layer, K | V, head): column col of the chosen clip into the prompt's other clips
__global__ void __launch_bounds__(128) cs_fork_kernel(CsArgs a, bf16* kcache, bf16* vcache, long long layer_elems,
                                                      int H, int s_max) {
  const int head = blockIdx.x % H, kv = (blockIdx.x / H) & 1, l = blockIdx.x / (2 * H);
  const int col = a.ctl[3] + a.ctl[0] + a.step, k = a.k;
  const long long clip_elems = (long long)H * s_max * 128;
  const bf16* base = (kv ? vcache : kcache) + l * layer_elems + (long long)head * s_max * 128 + (long long)col * 128;
  for (int e = threadIdx.x; e < a.B * k * 16; e += blockDim.x) {
    const int b = e / (k * 16), j = (e >> 4) % k, q = e & 15;
    const int js = a.chosen[b];
    if (j == js) continue;
    const uint4* src = reinterpret_cast<const uint4*>(base + cs_row(a, b, js) * clip_elems) + q;
    uint4* dst = reinterpret_cast<uint4*>(const_cast<bf16*>(base) + cs_row(a, b, j) * clip_elems) + q;
    *dst = *src;
  }
}

__global__ void __launch_bounds__(256) cs_norm_kernel(const bf16* ctx, float* norm, int rows, long long ctx_rows,
                                                      int D) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), b = blockIdx.y;
  if (r >= rows) return;
  const bf16* x = ctx + ((long long)b * ctx_rows + r) * D;
  const float n = sqrtf(warp_dot(x, x, D));
  if ((threadIdx.x & 31) == 0) norm[(long long)b * ctx_rows + r] = n;
}

}  // namespace

int launch_cs_candidates(const CsArgs& a, cudaStream_t stream) {
  VCL_REQUIRE(a.k >= 2 && a.k <= VCL_CS_MAX_K && a.B >= 1, "cs_candidates: k=%d outside 2..%d or B=%d", a.k,
              VCL_CS_MAX_K, a.B);
  VCL_REQUIRE(a.V >= a.k && a.V <= VCL_SAMPLE_WIDE_MAX_V && a.ld >= a.V, "cs_candidates: V=%d outside %d..%d or row "
              "pitch %lld < V", a.V, a.k, VCL_SAMPLE_WIDE_MAX_V, a.ld);
  static bool attr = false;
  if (!attr) {
    VCL_CUDA_OK(cudaFuncSetAttribute(cs_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     VCL_SAMPLE_WIDE_MAX_V * 4));
    attr = true;
  }
  cs_candidates_kernel<<<a.B, SEL_THREADS, ((size_t)a.V * 4 + 15) / 16 * 16, stream>>>(a);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_cs_rank(const CsArgs& a, cudaStream_t stream) {
  VCL_REQUIRE(a.k >= 2 && a.k <= VCL_CS_MAX_K && a.B >= 1, "cs_rank: k=%d outside 2..%d or B=%d", a.k, VCL_CS_MAX_K,
              a.B);
  VCL_REQUIRE(a.D >= 8 && a.D % 8 == 0 && a.D <= CS_MAX_D && a.ldh % 8 == 0, "cs_rank: D=%d must be a multiple of 8 "
              "up to %d (row pitch %lld)", a.D, CS_MAX_D, a.ldh);
  static bool attr = false;
  if (!attr) {
    VCL_CUDA_OK(cudaFuncSetAttribute(cs_sim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     CS_KG * CS_MAX_D * 2));
    attr = true;
  }
  cs_sim_kernel<<<dim3(CS_SPLIT, (a.k + CS_KG - 1) / CS_KG, a.B), 256, (size_t)CS_KG * a.D * 2, stream>>>(a);
  VCL_CUDA_OK(cudaGetLastError());
  cs_pick_kernel<<<a.B, 128, 0, stream>>>(a);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(2);
  return 0;
}

int launch_cs_fork(const CsArgs& a, bf16* kcache, bf16* vcache, long long layer_elems, int L, int H, int s_max,
                   cudaStream_t stream) {
  if (L == 0) return 0;
  cs_fork_kernel<<<L * 2 * H, 128, 0, stream>>>(a, kcache, vcache, layer_elems, H, s_max);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_cs_norms(const bf16* ctx, float* norm, int B, int rows, long long ctx_rows, int D, cudaStream_t stream) {
  VCL_REQUIRE(D >= 8 && D % 8 == 0 && rows >= 1 && rows <= ctx_rows, "cs_norms: D=%d, rows %d of %lld", D, rows,
              ctx_rows);
  cs_norm_kernel<<<dim3((rows + 7) / 8, B), 256, 0, stream>>>(ctx, norm, rows, ctx_rows, D);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

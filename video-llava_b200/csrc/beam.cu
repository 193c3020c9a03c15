// Beam search on the device: the per-step selection of transformers' _beam_search (greedy, do_sample=False) and
// the KV-cache forks it implies.
//
// Reference: video_chatgpt/inference.py:105-112 calls HF generate; generate(num_beams=k) runs _beam_search, whose
// step 1-3 this file restates (DESIGN.md section 3, "Beam search"):
//   lp_j     the greedy log-prob rule of the sampler, (x_j - m) - logf(W), on the beam's logits row (select.cuh's
//            kept_weights, so lp is vcl_op_sample_logprobs' value bit for bit; a row without a finite maximum is NaN)
//   key_j    fp32(lp_j + running score): selected on the summed key itself, since the add can create ties
//   top K    K = 2k of the k * V keys of an item, best first; ties go to the lowest flat index beam * V + token
//            (torch.topk leaves them unordered; this is our rule)
//   hit      token == eos, or t + 1 >= n_total (MaxLengthCriteria at cur_len + 1 = max_length)
//   running  the k best of key + hit * -1e9, ties to the lower candidate index
// Steps 4-6 (finished hypotheses, early stopping, output) run on the host from the records this file writes.
//
// beam_rows_kernel   one CTA per beam row: stage the 32-bit keys of x, m and W, rewrite them to keys of
//                    lp + score, collect the row's top K (radix select, select.cuh)
// beam_merge_kernel  one CTA per item: the item's top K of its k * K row candidates, hits, running picks, records,
//                    and (with a clip map) the slot assignment, next tokens and fork list
// kv_fork_kernel     the column copies of the forks
#include <math.h>

#include "common.cuh"
#include "kernels.h"
#include "select.cuh"

namespace vcl {

namespace {

constexpr int BM_MAX_K = 2 * VCL_BEAM_MAX;            // candidates per item
constexpr int BM_MAX_V = VCL_SAMPLE_WIDE_MAX_V;       // the staged row of 32-bit keys: 224 KB of shared memory

__global__ void __launch_bounds__(SEL_THREADS, 1) beam_rows_kernel(BeamArgs a) {
  extern __shared__ __align__(16) uint32_t skey[];
  __shared__ uint32_t s_max[SEL_WARPS];
  __shared__ float s_sum[SEL_WARPS];
  __shared__ uint32_t s_hist[256];
  __shared__ uint32_t s_wcnt[8];
  __shared__ uint32_t s_sel[2];
  __shared__ uint32_t s_cnt[SEL_WARPS];
  __shared__ int s_ntop;
  __shared__ uint32_t s_top_key[BM_MAX_K];
  __shared__ int s_top_idx[BM_MAX_K];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r = blockIdx.x, k = a.k, K = 2 * k, V = a.V;
  const int item = r / k, j = r - item * k;
  const int row = a.first ? item : (a.map != nullptr ? a.map[r] : r);
  const float* x = a.logits + (long long)row * a.ld;
  const float score = a.first ? (j == 0 ? 0.f : -1e9f) : a.score[r];

  // stage the keys of x and find the largest
  uint32_t best = 0;
  constexpr int U = 8;
  for (int i0 = tid; i0 < V; i0 += SEL_THREADS * U) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * SEL_THREADS;
      v[u] = i < V ? x[i] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * SEL_THREADS;
      if (i < V) {
        const uint32_t key = order_key32(v[u]);
        skey[i] = key;
        best = key > best ? key : best;
      }
    }
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

  // the greedy log-prob rule: lp_j = (x_j - m) - logf(W), W summed over every non-NaN token as the sampler does
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
  // rewrite each key as the key of fp32(lp_j + score); without a finite maximum every lp is NaN (key 0)
  for (int i = i_beg; i < i_end; ++i) {
    const float lp = __fsub_rn(__fsub_rn(key_value32(skey[i]), m), lw);
    skey[i] = finite ? order_key32(__fadd_rn(lp, score)) : 0u;
  }
  __syncthreads();
  collect_top<4>(skey, V, K, i_beg, i_end, s_hist, s_wcnt, s_sel, s_cnt, &s_ntop, s_top_key, s_top_idx);
  if (tid < K) {
    a.cand_key[(long long)r * K + tid] = s_top_key[tid];
    a.cand_tok[(long long)r * K + tid] = s_top_idx[tid];
  }
}

// (key desc, beam asc, token asc): the flat-index tie rule
__device__ __forceinline__ bool better(uint32_t ka, int ba, int ta, uint32_t kb, int bb, int tb) {
  return ka > kb || (ka == kb && (ba < bb || (ba == bb && ta < tb)));
}

__global__ void __launch_bounds__(BM_MAX_K * VCL_BEAM_MAX) beam_merge_kernel(BeamArgs a) {
  __shared__ uint32_t s_key[BM_MAX_K * VCL_BEAM_MAX];
  __shared__ int s_beam[BM_MAX_K * VCL_BEAM_MAX], s_tok[BM_MAX_K * VCL_BEAM_MAX];
  __shared__ uint32_t q_key[BM_MAX_K];
  __shared__ int q_beam[BM_MAX_K], q_tok[BM_MAX_K];
  // the serial tail's arrays (shared, not a local-memory stack frame)
  __shared__ float masked[BM_MAX_K];
  __shared__ int pick[VCL_BEAM_MAX], old[VCL_BEAM_MAX], nw[VCL_BEAM_MAX];
  const int tid = threadIdx.x, item = blockIdx.x, k = a.k, K = 2 * k, n = k * K;
  if (tid < n) {
    const int j = tid / K;
    const long long c = ((long long)item * k + j) * K + (tid - j * K);
    s_key[tid] = a.cand_key[c];
    s_beam[tid] = j;
    s_tok[tid] = a.cand_tok[c];
  }
  __syncthreads();
  if (tid < n) {   // the rank of this candidate among the item's k * K (all distinct by flat index)
    const uint32_t key = s_key[tid];
    const int b = s_beam[tid], t = s_tok[tid];
    int rank = 0;
    for (int c = 0; c < n; ++c) rank += better(s_key[c], s_beam[c], s_tok[c], key, b, t);
    if (rank < K) { q_key[rank] = key; q_beam[rank] = b; q_tok[rank] = t; }
  }
  __syncthreads();
  if (tid != 0) return;

  const int step = a.ctl[0] + a.step, n_total = a.ctl[1], eos = a.ctl[2];
  const bool last = step + 1 >= n_total;
  for (int q = 0; q < K; ++q) {
    const float s = key_value32(q_key[q]);
    const bool hit = last || (eos >= 0 && q_tok[q] == eos);
    masked[q] = __fadd_rn(s, hit ? -1e9f : -0.f);   // HF: score + hit.float() * -1e9
    a.rec[(long long)item * K + q] = BeamRec{s, q_beam[q], q_tok[q]};
  }
  // the running beams: the k best masked scores, ties to the lower index
  unsigned taken = 0;
  for (int r = 0; r < k; ++r) {
    int qb = -1;
    uint32_t kb = 0;
    for (int q = 0; q < K; ++q) {
      const uint32_t kq = order_key32(masked[q]);
      if (!((taken >> q) & 1u) && (qb < 0 || kq > kb)) { qb = q; kb = kq; }
    }
    taken |= 1u << qb;
    pick[r] = qb;
    a.pick[(long long)item * k + r] = qb;
  }
  for (int r = 0; r < k; ++r)
    if (a.score_out != nullptr) a.score_out[item * k + r] = masked[pick[r]];
  if (a.map == nullptr) {
    if (a.tok_out != nullptr)
      for (int r = 0; r < k; ++r) a.tok_out[item * k + r] = q_tok[pick[r]];
    return;
  }
  // slots: a parent keeps its clip for its first child; the other children take the clips of parents without one.
  // After the prefill every beam is the prompt, so every child counts as a child of beam 0 (the prompt's clip)
  unsigned used = 0;
  for (int j = 0; j < k; ++j) old[j] = a.map[item * k + j];
  for (int r = 0; r < k; ++r) {
    const int p = a.first ? 0 : q_beam[pick[r]];
    nw[r] = -1;
    if (!((used >> p) & 1u)) { used |= 1u << p; nw[r] = old[p]; }
  }
  int f = 0;
  for (int r = 0; r < k; ++r) {
    int2 fk = make_int2(-1, -1);
    if (nw[r] < 0) {
      while ((used >> f) & 1u) ++f;
      const int p = a.first ? 0 : q_beam[pick[r]];
      nw[r] = old[f++];
      fk = make_int2(old[p], nw[r]);
    }
    a.fork[item * k + r] = fk;
  }
  for (int r = 0; r < k; ++r) {
    a.map[item * k + r] = nw[r];
    a.tok_out[nw[r]] = q_tok[pick[r]];
  }
}

// one CTA per (layer, K | V, head): the forked column spans are contiguous ([s_max][128] per head)
__global__ void __launch_bounds__(256) kv_fork_kernel(bf16* kcache, bf16* vcache, long long layer_elems, int H,
                                                      int s_max, const int2* fork, int n, const int* ctl, int step,
                                                      int first) {
  const int head = blockIdx.x % H, kv = (blockIdx.x / H) & 1, l = blockIdx.x / (2 * H);
  const int S = ctl[3], t = ctl[0] + step;
  const int c0 = first ? 0 : S, c1 = S + t - 1;
  if (c1 < c0) return;
  const long long clip_elems = (long long)H * s_max * 128;
  bf16* base = (kv ? vcache : kcache) + l * layer_elems + (long long)head * s_max * 128 + (long long)c0 * 128;
  const int n16 = (c1 - c0 + 1) * 128 * 2 / 16;   // uint4 per span
  for (int e = 0; e < n; ++e) {
    const int2 fk = fork[e];
    if (fk.x < 0) continue;
    const uint4* src = reinterpret_cast<const uint4*>(base + fk.x * clip_elems);
    uint4* dst = reinterpret_cast<uint4*>(base + fk.y * clip_elems);
    for (int i = threadIdx.x; i < n16; i += blockDim.x) dst[i] = src[i];
  }
}

}  // namespace

int launch_beam_select(const BeamArgs& a, cudaStream_t stream) {
  VCL_REQUIRE(a.k >= 2 && a.k <= VCL_BEAM_MAX, "beam_select: k=%d outside 2..%d", a.k, VCL_BEAM_MAX);
  VCL_REQUIRE(a.V >= 2 * a.k && a.V <= BM_MAX_V && a.ld >= a.V, "beam_select: V=%d outside %d..%d or row pitch %lld < V",
              a.V, 2 * a.k, BM_MAX_V, a.ld);
  VCL_REQUIRE(a.B >= 1 && a.logits && a.ctl && a.rec && a.pick && a.cand_key && a.cand_tok &&
                  (a.first || a.score) && (a.map == nullptr || (a.tok_out && a.fork)),
              "beam_select: null argument");
  static bool attr = false;
  if (!attr) {
    VCL_CUDA_OK(cudaFuncSetAttribute(beam_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BM_MAX_V * 4));
    attr = true;
  }
  const size_t smem = ((size_t)a.V * 4 + 15) / 16 * 16;
  beam_rows_kernel<<<a.B * a.k, SEL_THREADS, smem, stream>>>(a);
  VCL_CUDA_OK(cudaGetLastError());
  beam_merge_kernel<<<a.B, BM_MAX_K * VCL_BEAM_MAX, 0, stream>>>(a);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(2);
  return 0;
}

int launch_kv_fork(bf16* kcache, bf16* vcache, long long layer_elems, int L, int H, int s_max, const int2* fork, int n,
                   const int* ctl, int step, int first, cudaStream_t stream) {
  if (L == 0) return 0;
  kv_fork_kernel<<<L * 2 * H, 256, 0, stream>>>(kcache, vcache, layer_elems, H, s_max, fork, n, ctl, step, first);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

// Classifier-free guidance of paired logits rows on the device, one CTA per pair.
//
// transformers' UnbatchedClassifierFreeGuidanceLogitsProcessor (generate(guidance_scale=g, negative_prompt_ids=...))
// runs an unconditional sequence next to every row and replaces the row's scores with
//   g * (log_softmax(cond) - log_softmax(uncond)) + log_softmax(uncond)
// Here the unconditional sequence is another clip of the cache: row b (guided) has partner row u, and the guidance
// table gives u (-1: row b is not guided) and g. The rule (DESIGN.md section 3, "Classifier-free guidance"), per row
// x of V fp32 logits, the whole computation in fp32 with no contraction:
//   m      the largest x_i; NaN when the row holds a NaN (torch's max propagates it)
//   S      sum of expf(x_i - m) over i, in one fixed order: thread t sums i = t, t + T, t + 2T, ... in rising i,
//          then a fixed xor tree inside each warp and the warp sums in warp order
//   l_i    (x_i - m) - logf(S)
//   out_i  g * (lc_i - lu_i) + lu_i   (lc of row b, lu of row u; the multiply and the add rounded apart)
// written over row b in place; row u is left alone. A row of NaN m or S (a NaN logit, every logit -inf, a +inf logit)
// gives NaN log-probs, and IEEE arithmetic takes it from there, as torch's fp32 formula does.
//
// The unconditional row is staged in shared memory (V * 4 bytes, V <= VCL_SAMPLE_WIDE_MAX_V); the conditional row
// comes from HBM once and its two later passes hit L2 (at V = 32 003 both rows are 256 KB, more than a CTA's shared
// memory).
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

constexpr int GD_THREADS = 1024;
constexpr int GD_WARPS = GD_THREADS / 32;

// the block-wide sum of v in the fixed order of the rule above; every thread gets it. s_red: GD_WARPS floats
__device__ __forceinline__ float block_sum(float v, float* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();   // s_red may still be read by an earlier call
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float t = s_red[0];
#pragma unroll
  for (int w = 1; w < GD_WARPS; ++w) t = __fadd_rn(t, s_red[w]);
  return t;
}

// the block-wide maximum with NaN propagated (flag: some thread saw a NaN); every thread gets it
__device__ __forceinline__ float block_max(float v, bool nan, float* s_red, int* s_nan) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();   // s_red / s_nan may still be read by an earlier call
  if (threadIdx.x == 0) *s_nan = 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  if (nan) *s_nan = 1;
  __syncthreads();
  float t = s_red[0];
#pragma unroll
  for (int w = 1; w < GD_WARPS; ++w) t = fmaxf(t, s_red[w]);
  return *s_nan ? __int_as_float(0x7fffffff) : t;
}

__global__ void __launch_bounds__(GD_THREADS, 1)
guidance_kernel(float* logits, long long ld, int B, int V, const int* __restrict__ partner,
                const float* __restrict__ scale) {
  extern __shared__ __align__(16) float s_u[];
  __shared__ float s_red[GD_WARPS];
  __shared__ int s_nan;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int u = partner[b];
  if (u < 0 || u >= B || u == b) return;   // (uniform over the CTA)
  const float g = scale[b];
  float* xc = logits + (long long)b * ld;
  const float* xu = logits + (long long)u * ld;

  float mc = -INFINITY, mu = -INFINITY;
  bool nc = false, nu = false;
  for (int i = tid; i < V; i += GD_THREADS) {
    const float c = xc[i], v = xu[i];
    s_u[i] = v;
    nc |= c != c; nu |= v != v;
    mc = fmaxf(mc, c); mu = fmaxf(mu, v);
  }
  mc = block_max(mc, nc, s_red, &s_nan);
  mu = block_max(mu, nu, s_red, &s_nan);

  float sc = 0.f, su = 0.f;
  for (int i = tid; i < V; i += GD_THREADS) {
    sc = __fadd_rn(sc, expf(__fsub_rn(xc[i], mc)));
    su = __fadd_rn(su, expf(__fsub_rn(s_u[i], mu)));
  }
  const float lsc = logf(block_sum(sc, s_red));
  const float lsu = logf(block_sum(su, s_red));

  for (int i = tid; i < V; i += GD_THREADS) {
    const float lc = __fsub_rn(__fsub_rn(xc[i], mc), lsc);
    const float lu = __fsub_rn(__fsub_rn(s_u[i], mu), lsu);
    xc[i] = __fadd_rn(__fmul_rn(g, __fsub_rn(lc, lu)), lu);
  }
}

// the token of every guided row b to its partner u: tok[u * stride] = tok[b * stride]. The next decode step's first
// kernel (launched with programmatic stream serialisation) may become resident meanwhile; it waits for this grid
// before it reads the tokens.
__global__ void guidance_handoff_kernel(int* tok, long long stride, int B, const int* __restrict__ partner) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int u = partner[b];
    if (u >= 0 && u < B && u != b) tok[(long long)u * stride] = tok[(long long)b * stride];
  }
}

}  // namespace

int launch_guidance(float* logits, long long ld, int B, int V, const int* partner, const float* scale,
                    cudaStream_t stream) {
  VCL_REQUIRE(V >= 1 && V <= VCL_SAMPLE_WIDE_MAX_V && ld >= V, "guidance: V=%d outside 1..%d or row pitch %lld < V",
              V, VCL_SAMPLE_WIDE_MAX_V, ld);
  VCL_REQUIRE(logits && partner && scale, "guidance: null argument");
  if (B <= 0) return 0;
  static bool attr = false;
  if (!attr) {
    VCL_CUDA_OK(cudaFuncSetAttribute(guidance_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     VCL_SAMPLE_WIDE_MAX_V * 4));
    attr = true;
  }
  guidance_kernel<<<B, GD_THREADS, (size_t)V * 4, stream>>>(logits, ld, B, V, partner, scale);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_guidance_handoff(int* tok, long long stride, int B, const int* partner, cudaStream_t stream) {
  if (B <= 0) return 0;
  guidance_handoff_kernel<<<1, 64, 0, stream>>>(tok, stride, B, partner);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

// Spatio-temporal mean pool: patch features [T, P, C] -> [n_temporal + P, C] video tokens.
//
// Reference: video_chatgpt/inference.py:13-44 (get_spatio_temporal_features_torch) and the numpy
// twin scripts/save_spatio_temporal_clip_features.py:46-57:
//   rows 0..T-1            mean over the P patches of frame t       ("temporal" tokens)
//   rows T..n_temporal-1   zeros (only when T < n_temporal)
//   rows n_temporal..      mean over the T frames of patch p        ("spatial" tokens)
// torch.mean accumulates in fp32 and rounds to the input dtype; the reference then casts the
// concatenation to fp16 (`.half()`), so the result is round_out(round_in(fp32 mean)).
//
// HBM-bound: 2*T*P*C bytes in, (n_temporal+P)*C*2 out (52.4 MB / 0.73 MB at T=100, P=256).
// One launch, two CTA roles, no atomics and a fixed summation order (deterministic):
//   blockIdx <  n_temporal   temporal role: CTA reduces the P patch rows of one frame
//   blockIdx >= n_temporal   spatial  role: CTA reduces the T frames of one patch row
// A CTA is 4 row groups x 64 lanes and owns ONE output row x 512 channels: a lane owns 8 consecutive
// channels (one coalesced 128-bit load per input row, 1 KB contiguous per group), the 4 groups deal the
// input rows round-robin with 8 loads in flight per lane, and a fixed-order shared-memory combine of the
// 4 partial sums finishes the mean (deterministic). 2 x 356 = 712 CTAs of 256 threads: ALL resident at
// once (one wave, ~5 per SM, ~150 KB of loads in flight per SM).
// Both roles stream the same tensor concurrently, so the second touch of a line is an L2 hit rather
// than a second HBM read.
#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

template <bool IN_BF16>
__device__ __forceinline__ void acc8(const uint4& u, float* a) {
  if (IN_BF16) {
    a[0] += bf16lo(u.x); a[1] += bf16hi(u.x); a[2] += bf16lo(u.y); a[3] += bf16hi(u.y);
    a[4] += bf16lo(u.z); a[5] += bf16hi(u.z); a[6] += bf16lo(u.w); a[7] += bf16hi(u.w);
  } else {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __half22float2(h[j]);
      a[2 * j] += f.x;
      a[2 * j + 1] += f.y;
    }
  }
}

template <bool IN_BF16, bool OUT_BF16>
__device__ __forceinline__ uint32_t round_pair(float x, float y) {
  // round to the input dtype first (torch.mean's result dtype), then to the output dtype
  if (IN_BF16) { x = bf16r(x); y = bf16r(y); }
  else { x = __half2float(__float2half_rn(x)); y = __half2float(__float2half_rn(y)); }
  if (OUT_BF16) return pack_bf16x2(x, y);
  __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<uint32_t*>(&h);
}

constexpr int POOL_GROUPS = 4;   // row groups per CTA (threadIdx.y)
constexpr int POOL_LANES = 64;   // lanes per group (threadIdx.x): 512 channels per CTA

template <bool IN_BF16, bool OUT_BF16>
__global__ void __launch_bounds__(POOL_LANES * POOL_GROUPS)
st_pool_kernel(const uint16_t* __restrict__ feats, long long frame_stride, long long patch_stride,
               int T, int P, int C, int n_temporal, uint16_t* __restrict__ out) {
  constexpr int UNROLL = 8;
  __shared__ float red[POOL_GROUPS][POOL_LANES * 8];
  const int g = threadIdx.y;
  const int c0 = (blockIdx.y * POOL_LANES + threadIdx.x) * 8;
  const bool c_ok = c0 < C;
  float a[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = 0.f;

  // One output row per CTA; its `n` input rows (stride `step`) are dealt round-robin to the 8
  // thread groups, each keeping UNROLL 128-bit loads in flight per thread.
  const int bid = blockIdx.x;
  const uint16_t* src = feats;
  long long step = 0;
  int n = 0;
  if (bid < n_temporal) {
    if (bid < T) { src = feats + (long long)bid * frame_stride; step = patch_stride; n = P; }
  } else {
    src = feats + (long long)(bid - n_temporal) * patch_stride; step = frame_stride; n = T;
  }
  if (c_ok) {
    src += c0;
    int r = g;
    for (; r + (UNROLL - 1) * POOL_GROUPS < n; r += UNROLL * POOL_GROUPS) {
      uint4 u[UNROLL];
#pragma unroll
      for (int k = 0; k < UNROLL; ++k) u[k] = ld_nc_v4(src + (long long)(r + k * POOL_GROUPS) * step);
#pragma unroll
      for (int k = 0; k < UNROLL; ++k) acc8<IN_BF16>(u[k], a);
    }
    for (; r < n; r += POOL_GROUPS) acc8<IN_BF16>(ld_nc_v4(src + (long long)r * step), a);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[g][threadIdx.x * 8 + j] = a[j];
  __syncthreads();
  if (g == 0 && c_ok) {
    // fixed-order combine of the 8 partial sums (deterministic), then the two roundings
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float s = red[0][threadIdx.x * 8 + j];
#pragma unroll
      for (int k = 1; k < POOL_GROUPS; ++k) s += red[k][threadIdx.x * 8 + j];
      a[j] = s;
    }
    const float denom = n > 0 ? (float)n : 1.f;   // n == 0: zero padding row
    uint4 o;
    o.x = round_pair<IN_BF16, OUT_BF16>(a[0] / denom, a[1] / denom);
    o.y = round_pair<IN_BF16, OUT_BF16>(a[2] / denom, a[3] / denom);
    o.z = round_pair<IN_BF16, OUT_BF16>(a[4] / denom, a[5] / denom);
    o.w = round_pair<IN_BF16, OUT_BF16>(a[6] / denom, a[7] / denom);
    *reinterpret_cast<uint4*>(out + (long long)bid * C + c0) = o;
  }
}

}  // namespace

int launch_st_pool(const void* feats, int in_dtype, long long frame_stride, long long patch_stride,
                   int T, int P, int C, int n_temporal, void* out, int out_dtype,
                   cudaStream_t stream) {
  VCL_REQUIRE(T >= 0 && P > 0 && C > 0 && n_temporal >= 0, "st_pool: bad shape T=%d P=%d C=%d", T, P, C);
  VCL_REQUIRE(T <= n_temporal, "st_pool: T=%d exceeds the %d temporal slots (the reference does not "
              "guard this; load_video never yields more)", T, n_temporal);
  VCL_REQUIRE(T > 0, "st_pool: T=0 would divide by zero in the spatial mean");
  VCL_REQUIRE(C % 8 == 0, "st_pool: C=%d must be a multiple of 8", C);
  VCL_REQUIRE(frame_stride % 8 == 0 && patch_stride % 8 == 0 && ((uintptr_t)feats % 16) == 0 &&
                  ((uintptr_t)out % 16) == 0, "st_pool: 16-byte alignment required");
  VCL_REQUIRE((in_dtype | 1) == 1 && (out_dtype | 1) == 1, "st_pool: dtype codes are 0=fp16 1=bf16");
  dim3 grid(n_temporal + P, (C / 8 + POOL_LANES - 1) / POOL_LANES);
  const uint16_t* f = reinterpret_cast<const uint16_t*>(feats);
  uint16_t* o = reinterpret_cast<uint16_t*>(out);
#define VCL_POOL(IB, OB) \
  st_pool_kernel<IB, OB><<<grid, dim3(POOL_LANES, POOL_GROUPS), 0, stream>>>(f, frame_stride, patch_stride, T, P, C, n_temporal, o)
  if (in_dtype == 1 && out_dtype == 1) VCL_POOL(true, true);
  else if (in_dtype == 1 && out_dtype == 0) VCL_POOL(true, false);
  else if (in_dtype == 0 && out_dtype == 1) VCL_POOL(false, true);
  else VCL_POOL(false, false);
#undef VCL_POOL
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

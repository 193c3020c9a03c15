// Cross-entropy over bf16 logits: per-row NLL, the mean loss, and an optional compact copy of the logits.
//
// Reference: video_chatgpt/model/video_chatgpt.py:225-239, lm_head over every position, then
// CrossEntropyLoss on logits[..., :-1, :] against labels[..., 1:] (ignore_index -100). On bf16 logits
// torch computes log_softmax in fp32 (row max, then sum of exp(x - max), then x - max - log(sum)) and
// rounds it to bf16; nll_loss then negates the bf16 value at the label and averages in fp32. The rounding
// points here are the same:
//   nll[row] = -bf16((x[label] - max) - log(sum exp(x - max)))      (fp32 arithmetic)
// A row whose label is -100, or which has no target, gives 0 and is not counted; a label outside
// 0 .. V-1 gives NaN (it is never used as an index).
//
// HBM-bound: the logits are read once (29 MB for 448 rows of 32 003). One CTA of 256 threads per row: it
// stages the row in shared memory with 16-byte loads (4 in flight per thread), reduces the maximum, sums the
// exponentials from shared memory and, when asked, writes the compact [rows, V] copy from shared memory with
// 16-byte stores aligned to the destination. A second kernel (one CTA) takes the mean over the counted rows in
// a fixed order (fp64 accumulation, no atomics), so the loss is identical from run to run.
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

constexpr int CE_THREADS = 256;
constexpr int CE_UNROLL = 4;
constexpr int CE_MAX_SMEM = 160 * 1024;   // the staged row: V <= 81 920
constexpr int MEAN_THREADS = 512;

// label of row r: labels[r] (seg == 0), or the HF shift over clips of seg columns (row r = clip r / seg,
// column r % seg is scored against column r % seg + 1; the last column has no target). -100: not scored.
__device__ __forceinline__ long long target_of(const long long* labels, long long r, int seg) {
  if (seg == 0) return labels[r];
  return (r % seg == seg - 1) ? -100ll : labels[r + 1];
}

__global__ void __launch_bounds__(CE_THREADS)
cross_entropy_rows_kernel(const uint16_t* __restrict__ logits, long long ld, int V, const long long* __restrict__ labels,
                          long long row0, int seg, float* __restrict__ nll, uint16_t* __restrict__ logits_out) {
  extern __shared__ __align__(16) uint16_t srow[];
  __shared__ float red[CE_THREADS / 32];
  const int tid = threadIdx.x;
  const long long r = blockIdx.x;
  const uint16_t* x = logits + r * ld;
  const int n8 = V / 8;

  // stage the row, keeping the maximum
  float mx = -INFINITY;
  for (int c0 = tid; c0 < n8; c0 += CE_THREADS * CE_UNROLL) {
    uint4 u[CE_UNROLL];
#pragma unroll
    for (int k = 0; k < CE_UNROLL; ++k) {
      const int c = c0 + k * CE_THREADS;
      if (c < n8) u[k] = ld_nc_v4(x + (long long)c * 8);
    }
#pragma unroll
    for (int k = 0; k < CE_UNROLL; ++k) {
      const int c = c0 + k * CE_THREADS;
      if (c < n8) {
        *reinterpret_cast<uint4*>(srow + c * 8) = u[k];
        mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(bf16lo(u[k].x), bf16hi(u[k].x)), fmaxf(bf16lo(u[k].y), bf16hi(u[k].y))),
                             fmaxf(fmaxf(bf16lo(u[k].z), bf16hi(u[k].z)), fmaxf(bf16lo(u[k].w), bf16hi(u[k].w)))));
      }
    }
  }
  for (int i = n8 * 8 + tid; i < V; i += CE_THREADS) {
    srow[i] = x[i];
    mx = fmaxf(mx, __uint_as_float((uint32_t)srow[i] << 16));
  }
  mx = warp_max(mx);
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < CE_THREADS / 32; ++w) mx = fmaxf(mx, red[w]);

  // sum of exp(x - max) over the staged row (each thread re-reads the chunks it wrote)
  float s = 0.f;
  for (int c = tid; c < n8; c += CE_THREADS) {
    const uint4 u = *reinterpret_cast<const uint4*>(srow + c * 8);
    s += expf(bf16lo(u.x) - mx) + expf(bf16hi(u.x) - mx) + expf(bf16lo(u.y) - mx) + expf(bf16hi(u.y) - mx) +
         expf(bf16lo(u.z) - mx) + expf(bf16hi(u.z) - mx) + expf(bf16lo(u.w) - mx) + expf(bf16hi(u.w) - mx);
  }
  for (int i = n8 * 8 + tid; i < V; i += CE_THREADS) s += expf(__uint_as_float((uint32_t)srow[i] << 16) - mx);
  s = warp_sum(s);
  __syncthreads();                       // every thread has read red[] (the maximum) before it is reused
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();

  if (tid == 0 && nll != nullptr) {
    float sum = red[0];
#pragma unroll
    for (int w = 1; w < CE_THREADS / 32; ++w) sum += red[w];
    const long long t = target_of(labels, row0 + r, seg);
    float v = 0.f;
    if (t != -100) {
      if (t < 0 || t >= V) {
        v = __int_as_float(0x7fc00000);   // NaN
      } else {
        const float xt = __uint_as_float((uint32_t)srow[t] << 16);
        v = -bf16r((xt - mx) - logf(sum));
      }
    }
    nll[r] = v;
  }

  if (logits_out != nullptr) {
    // compact copy: the destination row starts at any 2-byte boundary; peel to 16-byte alignment
    uint16_t* o = logits_out + r * V;
    int h0 = (int)(((16u - ((uint32_t)(uintptr_t)o & 15u)) & 15u) >> 1);
    if (h0 > V) h0 = V;
    const int nv = (V - h0) / 8;
    for (int i = tid; i < h0; i += CE_THREADS) o[i] = srow[i];
    for (int c = tid; c < nv; c += CE_THREADS) {
      const uint16_t* p = srow + h0 + c * 8;
      uint4 w;
      w.x = p[0] | ((uint32_t)p[1] << 16); w.y = p[2] | ((uint32_t)p[3] << 16);
      w.z = p[4] | ((uint32_t)p[5] << 16); w.w = p[6] | ((uint32_t)p[7] << 16);
      *reinterpret_cast<uint4*>(o + h0 + c * 8) = w;
    }
    for (int i = h0 + nv * 8 + tid; i < V; i += CE_THREADS) o[i] = srow[i];
  }
}

// mean of nll over the counted rows (fixed order: per-thread strided sums, then a fixed tree), and the copy of
// the scored rows into nll_out ([clip][seg - 1] with a shift; [rows] otherwise, skipped when it is nll itself)
__global__ void __launch_bounds__(MEAN_THREADS)
nll_mean_kernel(const float* __restrict__ nll, const long long* __restrict__ labels, long long rows, int seg,
                float* nll_out, float* loss_out) {
  __shared__ double ssum[MEAN_THREADS];
  __shared__ long long scnt[MEAN_THREADS];
  const int tid = threadIdx.x;
  double sum = 0.0;
  long long cnt = 0;
  for (long long r = tid; r < rows; r += MEAN_THREADS) {
    const float v = nll[r];
    if (target_of(labels, r, seg) != -100) {
      sum += (double)v;
      ++cnt;
    }
    if (nll_out != nullptr && nll_out != nll) {
      if (seg == 0) nll_out[r] = v;
      else if (r % seg != seg - 1) nll_out[r - r / seg] = v;
    }
  }
  ssum[tid] = sum;
  scnt[tid] = cnt;
  __syncthreads();
  for (int w = MEAN_THREADS / 2; w > 0; w >>= 1) {
    if (tid < w) {
      ssum[tid] += ssum[tid + w];
      scnt[tid] += scnt[tid + w];
    }
    __syncthreads();
  }
  if (tid == 0 && loss_out != nullptr)
    *loss_out = scnt[0] > 0 ? (float)(ssum[0] / (double)scnt[0]) : __int_as_float(0x7fc00000);
}

}  // namespace

int launch_cross_entropy(const bf16* logits, long long ld, int V, const long long* labels, long long row0, int rows,
                         int seg, float* nll, bf16* logits_out, cudaStream_t stream) {
  VCL_REQUIRE(V > 0 && rows >= 0 && seg >= 0 && row0 >= 0, "cross_entropy: bad shape V=%d rows=%d", V, rows);
  VCL_REQUIRE(ld >= V && ld % 8 == 0 && ((uintptr_t)logits % 16) == 0,
              "cross_entropy: logits need a 16-byte aligned base and a row pitch >= V that is a multiple of 8 "
              "(V=%d, ld=%lld)", V, ld);
  VCL_REQUIRE(((uintptr_t)logits_out % 2) == 0, "cross_entropy: logits_out must be 2-byte aligned");
  VCL_REQUIRE(nll == nullptr || labels != nullptr, "cross_entropy: nll needs labels");
  const size_t smem = ((size_t)V + 7) / 8 * 16;
  VCL_REQUIRE(smem <= (size_t)CE_MAX_SMEM, "cross_entropy: V=%d exceeds the staged row (at most %d columns)", V,
              CE_MAX_SMEM / 2);
  if (rows == 0) return 0;
  static bool attr = false;
  if (!attr) {
    VCL_CUDA_OK(cudaFuncSetAttribute(cross_entropy_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     CE_MAX_SMEM));
    attr = true;
  }
  cross_entropy_rows_kernel<<<rows, CE_THREADS, smem, stream>>>(
      reinterpret_cast<const uint16_t*>(logits), ld, V, labels, row0, seg, nll,
      reinterpret_cast<uint16_t*>(logits_out));
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_nll_mean(const float* nll, const long long* labels, long long rows, int seg, float* nll_out,
                    float* loss_out, cudaStream_t stream) {
  VCL_REQUIRE(nll != nullptr && labels != nullptr && rows >= 0 && seg >= 0, "nll_mean: bad arguments");
  if (nll_out == nullptr && loss_out == nullptr) return 0;
  nll_mean_kernel<<<1, MEAN_THREADS, 0, stream>>>(nll, labels, rows, seg, nll_out, loss_out);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

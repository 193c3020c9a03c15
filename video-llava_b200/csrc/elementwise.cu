// HBM-bound row-wise / elementwise kernels of the hot path: LayerNorm, RMSNorm, im2col for the
// patch-embed GEMM, CLIP embedding assembly + pre-LN, token-embedding gather with the video splice,
// RoPE + KV-cache write, arg-max. All use 128-bit accesses along the contiguous (channel) axis.
//
// Reference semantics followed (cited per kernel):
//   CLIP embeddings        transformers/models/clip/modeling_clip.py:138-218 (cat CLS, + pos)
//   CLIP pre_layrnorm      transformers/models/clip/modeling_clip.py:677
//   LlamaRMSNorm           transformers/models/llama/modeling_llama.py:53-67
//   RoPE                   transformers/models/llama/modeling_llama.py:124-168
//   embedding splice       video_chatgpt/model/video_chatgpt.py:100-168 (start/end-token branch)
#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

constexpr int NORM_THREADS = 128;
constexpr int NORM_MAXC = 8;  // 8 chunks x 8 elements x 128 threads = 8192 columns max

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  f[0] = bf16lo(u.x); f[1] = bf16hi(u.x); f[2] = bf16lo(u.y); f[3] = bf16hi(u.y);
  f[4] = bf16lo(u.z); f[5] = bf16hi(u.z); f[6] = bf16lo(u.w); f[7] = bf16hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
  return o;
}

__device__ __forceinline__ float block_sum_128(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // protect red[] from the previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  return red[0] + red[1] + red[2] + red[3];
}

// Normalise the row held in v[][] (fp32) and store bf16. RMS: y = w * bf16(x * rstd).
// LN: y = (x - mean) * rstd * w + b, one rounding.
template <bool RMS>
__device__ __forceinline__ void norm_store(float (&v)[NORM_MAXC][8], int nch, int D, bf16* y,
                                           const bf16* __restrict__ w, const bf16* __restrict__ b,
                                           float eps, float* red) {
  const int tid = threadIdx.x;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NORM_MAXC; ++i) {
    if (tid + i * NORM_THREADS < nch) {
#pragma unroll
      for (int j = 0; j < 8; ++j) s += RMS ? v[i][j] * v[i][j] : v[i][j];
    }
  }
  s = block_sum_128(s, red);
  float mean = 0.f, rstd;
  if (RMS) {
    rstd = rsqrtf(s / (float)D + eps);
  } else {
    mean = s / (float)D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NORM_MAXC; ++i) {
      if (tid + i * NORM_THREADS < nch) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q += d * d; }
      }
    }
    q = block_sum_128(q, red);
    rstd = rsqrtf(q / (float)D + eps);
  }
#pragma unroll
  for (int i = 0; i < NORM_MAXC; ++i) {
    const int c = tid + i * NORM_THREADS;
    if (c < nch) {
      float wv[8], o[8];
      unpack8(*reinterpret_cast<const uint4*>(w + c * 8), wv);
      if (RMS) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = wv[j] * bf16r(v[i][j] * rstd);
      } else {
        float bv[8];
        unpack8(*reinterpret_cast<const uint4*>(b + c * 8), bv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * wv[j] + bv[j];
      }
      *reinterpret_cast<uint4*>(y + c * 8) = pack8(o);
    }
  }
}

template <bool RMS>
__global__ void __launch_bounds__(NORM_THREADS)
rownorm_kernel(const bf16* __restrict__ x, long long ldx, bf16* __restrict__ y, long long ldy,
               const bf16* __restrict__ w, const bf16* __restrict__ b, int D, float eps) {
  __shared__ float red[4];
  const long long row = blockIdx.x;
  const int nch = D >> 3;
  float v[NORM_MAXC][8];
  const bf16* xr = x + row * ldx;
#pragma unroll
  for (int i = 0; i < NORM_MAXC; ++i) {
    const int c = threadIdx.x + i * NORM_THREADS;
    if (c < nch) unpack8(*reinterpret_cast<const uint4*>(xr + c * 8), v[i]);
  }
  norm_store<RMS>(v, nch, D, y + row * ldy, w, b, eps, red);
}

// Warp-per-row normalisation for the widths on the hot path (D = 256*CPL): every lane owns CPL
// 16-byte chunks of a row, a warp normalises ROWS rows at once (ROWS*CPL loads in flight per lane),
// statistics need only shuffles, and a CTA of 8 warps covers 8*ROWS rows. ~HBM speed.
template <bool RMS, int CPL, int ROWS>
__global__ void __launch_bounds__(256)
rownorm_warp_kernel(const bf16* __restrict__ x, long long ldx, bf16* __restrict__ y, long long ldy,
                    const bf16* __restrict__ w, const bf16* __restrict__ b, int rows, float eps) {
  constexpr int D = CPL * 256;
  // a following kernel launched with programmatic stream serialisation (the decode GEMVs) may become
  // resident and prefetch its weights while the rows are normalised; it waits for this grid's completion
  // (griddepcontrol.wait) before it reads them. No effect for ordinary successors.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int lane = threadIdx.x & 31;
  const long long row0 = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * ROWS;
  if (row0 >= rows) return;
  uint4 u[ROWS][CPL];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const long long row = row0 + r < rows ? row0 + r : rows - 1;
#pragma unroll
    for (int i = 0; i < CPL; ++i) u[r][i] = ld_nc_v4(x + row * ldx + (i * 32 + lane) * 8);
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    if (row0 + r >= rows) break;
    float v[CPL][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < CPL; ++i) {
      unpack8(u[r][i], v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += RMS ? v[i][j] * v[i][j] : v[i][j];
    }
    s = warp_sum(s);
    float mean = 0.f, rstd;
    if (RMS) {
      rstd = rsqrtf(s / (float)D + eps);
    } else {
      mean = s / (float)D;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < CPL; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q += d * d; }
      q = warp_sum(q);
      rstd = rsqrtf(q / (float)D + eps);
    }
    bf16* yr = y + (row0 + r) * ldy;
#pragma unroll
    for (int i = 0; i < CPL; ++i) {
      const int c = i * 32 + lane;
      float wv[8], o[8];
      unpack8(*reinterpret_cast<const uint4*>(w + c * 8), wv);
      if (RMS) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = wv[j] * bf16r(v[i][j] * rstd);
      } else {
        float bv[8];
        unpack8(*reinterpret_cast<const uint4*>(b + c * 8), bv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * wv[j] + bv[j];
      }
      *reinterpret_cast<uint4*>(yr + c * 8) = pack8(o);
    }
  }
}

template <bool RMS, int CPL, int ROWS>
void launch_rownorm_warp(const bf16* x, long long ldx, bf16* y, long long ldy, const bf16* w,
                         const bf16* b, int rows, float eps, cudaStream_t stream) {
  const int per_cta = 8 * ROWS;
  rownorm_warp_kernel<RMS, CPL, ROWS><<<(rows + per_cta - 1) / per_cta, 256, 0, stream>>>(x, ldx, y, ldy, w, b,
                                                                                            rows, eps);
}

__global__ void __launch_bounds__(NORM_THREADS)
clip_embed_ln_kernel(const bf16* __restrict__ patch_out, const bf16* __restrict__ cls,
                     const bf16* __restrict__ pos, const bf16* __restrict__ ln_w,
                     const bf16* __restrict__ ln_b, bf16* __restrict__ h, int P, int D, float eps) {
  __shared__ float red[4];
  const long long row = blockIdx.x;          // n * (P+1) + t
  const int t = (int)(row % (P + 1));
  const long long n = row / (P + 1);
  const int nch = D >> 3;
  const bf16* src = (t == 0) ? cls : patch_out + (n * P + (t - 1)) * (long long)D;
  const bf16* pr = pos + (long long)t * D;
  float v[NORM_MAXC][8];
#pragma unroll
  for (int i = 0; i < NORM_MAXC; ++i) {
    const int c = threadIdx.x + i * NORM_THREADS;
    if (c < nch) {
      float a[8], p[8];
      unpack8(*reinterpret_cast<const uint4*>(src + c * 8), a);
      unpack8(*reinterpret_cast<const uint4*>(pr + c * 8), p);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = bf16r(a[j] + p[j]);  // embeddings tensor is bf16
    }
  }
  norm_store<false>(v, nch, D, h + row * D, ln_w, ln_b, eps, red);
}

// One CTA per (frame, patch-row): reads `patch` image rows x 3 channels, scatters them into the
// G patches of that row. Source reads are fully coalesced.
__global__ void __launch_bounds__(256)
im2col_kernel(const void* __restrict__ pixels, int mode, bf16* __restrict__ out, int image,
              int patch, int KP) {
  const int G = image / patch;
  const int n = blockIdx.x / G, py = blockIdx.x % G;
  const int P = G * G;
  const int pp = patch * patch;
  const long long row0 = (long long)n * P + (long long)py * G;
  const int total = 3 * patch * image;
  if (mode == 0) {
    const bf16* src = reinterpret_cast<const bf16*>(pixels) + (long long)n * 3 * image * image;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
      const int c = e / (patch * image);
      const int r = e - c * patch * image;
      const int i = r / image, x = r - i * image;
      const int px = x / patch, j = x - px * patch;
      out[(row0 + px) * KP + c * pp + i * patch + j] =
          src[((long long)c * image + (py * patch + i)) * image + x];
    }
  } else {
    // uint8 NHWC; CLIPImageProcessor constants (transformers/models/clip/image_processing_clip.py)
    const float mean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
    const float stdv[3] = {0.26862954f, 0.26130258f, 0.27577711f};
    const uint8_t* src = reinterpret_cast<const uint8_t*>(pixels) +
                         ((long long)n * image + (long long)py * patch) * image * 3;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
      const int i = e / (image * 3);
      const int r = e - i * image * 3;
      const int x = r / 3, c = r - x * 3;
      const int px = x / patch, j = x - px * patch;
      const float val = ((float)src[e] * (1.0f / 255.0f) - mean[c]) / stdv[c];
      out[(row0 + px) * KP + c * pp + i * patch + j] = __float2bfloat16_rn(val);
    }
  }
  const int padw = KP - 3 * pp;
  for (int e = threadIdx.x; e < G * padw; e += blockDim.x) {
    const int px = e / padw, j = e - px * padw;
    out[(row0 + px) * KP + 3 * pp + j] = __float2bfloat16_rn(0.f);
  }
}

__global__ void __launch_bounds__(128)
embed_splice_kernel(const long long* __restrict__ ids, const bf16* __restrict__ table,
                    const bf16* __restrict__ vid, const int* __restrict__ vid_start,
                    bf16* __restrict__ h, int S, int D, int n_vid, int vocab, const int* __restrict__ pack) {
  const long long row = blockIdx.x;
  int b, s;
  if (pack != nullptr) {
    b = __ldg(pack_row(pack, row)); s = __ldg(pack_row(pack, row) + 1);
  } else {
    b = (int)(row / S); s = (int)(row % S);
  }
  // vid_start[b] = index of the row AFTER which the video rows go (-1: the video rows start at row 0);
  // anything below -1 (VCL_NO_VIDEO), or a null array, marks a text-only row
  const int vs = vid_start != nullptr ? vid_start[b] : -2;
  const bf16* src;
  if (vs >= -1 && s > vs && s <= vs + n_vid) {
    src = vid + ((long long)b * n_vid + (s - vs - 1)) * D;
  } else {
    long long id = ids[row];
    if (id < 0) id = 0;
    if (id >= vocab) id = vocab - 1;
    src = table + id * D;
  }
  bf16* dst = h + row * D;
  for (int c = threadIdx.x; c < (D >> 3); c += blockDim.x)
    *reinterpret_cast<uint4*>(dst + c * 8) = *reinterpret_cast<const uint4*>(src + c * 8);
}

__global__ void __launch_bounds__(128)
embed_tokens_kernel(const int* __restrict__ tok, long long tok_stride, const bf16* __restrict__ table,
                    bf16* __restrict__ h, int D, int vocab) {
  int id = tok[(long long)blockIdx.x * tok_stride];
  if (id < 0) id = 0;
  if (id >= vocab) id = vocab - 1;
  const bf16* src = table + (long long)id * D;
  bf16* dst = h + (long long)blockIdx.x * D;
  for (int c = threadIdx.x; c < (D >> 3); c += blockDim.x)
    *reinterpret_cast<uint4*>(dst + c * 8) = *reinterpret_cast<const uint4*>(src + c * 8);
}

__global__ void rope_table_kernel(bf16* cos_t, bf16* sin_t, int max_pos, int head_dim, float theta) {
  const int half = head_dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= max_pos * half) return;
  const int p = idx / half, i = idx - p * half;
  // inv_freq = 1 / theta^(2i/dim) in fp32, angle = pos * inv_freq in fp32, then cast to bf16
  const float inv = 1.0f / powf(theta, (float)(2 * i) / (float)head_dim);
  const float ang = (float)p * inv;
  cos_t[idx] = __float2bfloat16_rn(cosf(ang));
  sin_t[idx] = __float2bfloat16_rn(sinf(ang));
}

// One warp per (token, head); head_dim = 128. lanes 0-7: q pairs, 8-15: k pairs, 16-31: v copy.
__global__ void __launch_bounds__(256)
rope_kv_prefill_kernel(bf16* qkv, bf16* __restrict__ kcache, bf16* __restrict__ vcache,
                       const bf16* __restrict__ cos_t, const bf16* __restrict__ sin_t, int B, int S,
                       int H, int s_max, int pos0, const int* __restrict__ pos_dev,
                       const int* __restrict__ n_pad) {
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= (long long)B * S * H) return;
  const int head = (int)(wid % H);
  const long long tok = wid / H;
  const int b = (int)(tok / S), s = (int)(tok % S);
  const int D = H * 128;
  bf16* row = qkv + tok * 3LL * D;
  const int pos = pos0 + s + (pos_dev != nullptr ? __ldg(pos_dev + b) : 0);
  const long long cache_off = (((long long)b * H + head) * s_max + pos) * 128;
  // RoPE position of this cache column: left padding shifts it (pad columns clamp at 0)
  const int rpos = n_pad != nullptr ? max(pos - __ldg(n_pad + b), 0) : pos;
  if (lane < 16) {
    const int which = lane >> 3;              // 0 = q, 1 = k
    const int d0 = (lane & 7) * 8;            // 0..56, partner at +64
    bf16* base = row + (long long)which * D + head * 128;
    float lo[8], hi[8], c[8], sn[8], olo[8], ohi[8];
    unpack8(*reinterpret_cast<const uint4*>(base + d0), lo);
    unpack8(*reinterpret_cast<const uint4*>(base + d0 + 64), hi);
    unpack8(*reinterpret_cast<const uint4*>(cos_t + (long long)rpos * 64 + d0), c);
    unpack8(*reinterpret_cast<const uint4*>(sin_t + (long long)rpos * 64 + d0), sn);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // q*cos + rotate_half(q)*sin with every product and the sum rounded to bf16
      olo[j] = bf16r(lo[j] * c[j]) + bf16r(-hi[j] * sn[j]);
      ohi[j] = bf16r(hi[j] * c[j]) + bf16r(lo[j] * sn[j]);
    }
    const uint4 plo = pack8(olo), phi = pack8(ohi);
    if (which == 0) {
      *reinterpret_cast<uint4*>(base + d0) = plo;
      *reinterpret_cast<uint4*>(base + d0 + 64) = phi;
    } else {
      *reinterpret_cast<uint4*>(kcache + cache_off + d0) = plo;
      *reinterpret_cast<uint4*>(kcache + cache_off + d0 + 64) = phi;
    }
  } else {
    const int d0 = (lane - 16) * 8;
    *reinterpret_cast<uint4*>(vcache + cache_off + d0) =
        *reinterpret_cast<const uint4*>(row + 2LL * D + head * 128 + d0);
  }
}

__global__ void __launch_bounds__(1024)
argmax_kernel(const float* __restrict__ logits, int* __restrict__ out, long long out_stride, int V) {
  __shared__ float sv[32];
  __shared__ int si[32];
  const float* l = logits + (long long)blockIdx.x * V;
  // start at index 0, as torch.argmax does: a row with no logit above -inf (all -inf or NaN) gives token 0, a
  // valid row of the embedding table, instead of an index past the vocabulary
  float best = -INFINITY;
  int bi = 0;
  constexpr int U = 8;
  for (int i0 = threadIdx.x; i0 < V; i0 += 1024 * U) {
    float x[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * 1024;
      x[u] = (i < V) ? l[i] : -INFINITY;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * 1024;      // increasing index: ties keep the lowest
      if (x[u] > best) { best = x[u]; bi = i; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sv[warp] = best; si[warp] = bi; }
  __syncthreads();
  if (warp == 0) {
    best = sv[lane]; bi = si[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) out[(long long)blockIdx.x * out_stride] = bi;
  }
}

}  // namespace

int launch_layernorm(const bf16* x, long long ldx, bf16* y, long long ldy, const bf16* w,
                     const bf16* b, int rows, int D, float eps, cudaStream_t stream) {
  VCL_REQUIRE(D % 8 == 0 && D <= NORM_MAXC * 8 * NORM_THREADS, "layernorm: unsupported D=%d", D);
  VCL_REQUIRE(ldx % 8 == 0 && ldy % 8 == 0, "layernorm: pitches must be x8");
  if (rows <= 0) return 0;
  if (D == 1024) launch_rownorm_warp<false, 4, 2>(x, ldx, y, ldy, w, b, rows, eps, stream);
  else rownorm_kernel<false><<<rows, NORM_THREADS, 0, stream>>>(x, ldx, y, ldy, w, b, D, eps);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_rmsnorm(const bf16* x, long long ldx, bf16* y, long long ldy, const bf16* w, int rows,
                   int D, float eps, cudaStream_t stream) {
  VCL_REQUIRE(D % 8 == 0 && D <= NORM_MAXC * 8 * NORM_THREADS, "rmsnorm: unsupported D=%d", D);
  VCL_REQUIRE(ldx % 8 == 0 && ldy % 8 == 0, "rmsnorm: pitches must be x8");
  if (rows <= 0) return 0;
  if (D == 4096) launch_rownorm_warp<true, 16, 1>(x, ldx, y, ldy, w, nullptr, rows, eps, stream);
  else if (D == 5120) launch_rownorm_warp<true, 20, 1>(x, ldx, y, ldy, w, nullptr, rows, eps, stream);
  else rownorm_kernel<true><<<rows, NORM_THREADS, 0, stream>>>(x, ldx, y, ldy, w, nullptr, D, eps);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_im2col(const void* pixels, int mode, bf16* out, int n_frames, int image, int patch,
                  int KP, cudaStream_t stream) {
  VCL_REQUIRE(image % patch == 0 && KP >= 3 * patch * patch, "im2col: bad geometry");
  VCL_REQUIRE(mode == 0 || mode == 1, "im2col: mode must be 0 (bf16 NCHW) or 1 (uint8 NHWC)");
  if (n_frames <= 0) return 0;
  im2col_kernel<<<n_frames * (image / patch), 256, 0, stream>>>(pixels, mode, out, image, patch, KP);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_clip_embed_ln(const bf16* patch_out, const bf16* cls, const bf16* pos, const bf16* ln_w,
                         const bf16* ln_b, bf16* h, int n_frames, int P, int D, float eps,
                         cudaStream_t stream) {
  VCL_REQUIRE(D % 8 == 0 && D <= NORM_MAXC * 8 * NORM_THREADS, "clip_embed: unsupported D=%d", D);
  if (n_frames <= 0) return 0;
  clip_embed_ln_kernel<<<n_frames * (P + 1), NORM_THREADS, 0, stream>>>(patch_out, cls, pos, ln_w,
                                                                        ln_b, h, P, D, eps);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_embed_splice(const long long* ids, const bf16* table, const bf16* vid,
                        const int* vid_start, bf16* h, int B, int S, int D, int n_vid, int vocab,
                        cudaStream_t stream, const int* pack, int M) {
  VCL_REQUIRE(D % 8 == 0, "embed_splice: D must be x8");
  const int rows = pack != nullptr ? M : B * S;
  if (rows <= 0) return 0;
  embed_splice_kernel<<<rows, 128, 0, stream>>>(ids, table, vid, vid_start, h, S, D, n_vid, vocab, pack);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_embed_tokens(const int* tok, long long tok_stride, const bf16* table, bf16* h, int B,
                        int D, int vocab, cudaStream_t stream) {
  VCL_REQUIRE(D % 8 == 0, "embed_tokens: D must be x8");
  if (B <= 0) return 0;
  embed_tokens_kernel<<<B, 128, 0, stream>>>(tok, tok_stride, table, h, D, vocab);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_rope_table(bf16* cos_t, bf16* sin_t, int max_pos, int head_dim, float theta,
                      cudaStream_t stream) {
  const int n = max_pos * (head_dim / 2);
  rope_table_kernel<<<(n + 255) / 256, 256, 0, stream>>>(cos_t, sin_t, max_pos, head_dim, theta);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_rope_kv_prefill(bf16* qkv, bf16* kcache, bf16* vcache, const bf16* cos_t,
                           const bf16* sin_t, int B, int S, int H, int head_dim, int s_max, int pos0,
                           cudaStream_t stream, const int* pos_dev, const int* n_pad) {
  VCL_REQUIRE(head_dim == 128, "rope: head_dim must be 128 (got %d)", head_dim);
  VCL_REQUIRE(pos0 + S <= s_max, "rope: positions %d..%d exceed the cache (%d)", pos0, pos0 + S, s_max);
  const long long warps = (long long)B * S * H;
  if (warps <= 0) return 0;
  rope_kv_prefill_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(qkv, kcache, vcache, cos_t,
                                                                        sin_t, B, S, H, s_max, pos0, pos_dev, n_pad);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

__global__ void fill_int_kernel(int* dst, int value, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = value;
}

// Decode-path RMSNorm for 5..16 clips: one CTA per clip, output in the window-major layout the wide GEMV
// streams (kernels.h: xwin). w == null: plain re-layout.
__global__ void __launch_bounds__(256)
xwin_norm_kernel(const bf16* __restrict__ x, long long ldx, bf16* __restrict__ y, const bf16* __restrict__ w, int K,
                 float eps) {
  __shared__ float red[8];
  // the GEMV that follows may become resident and prefetch its weights meanwhile (it waits for this grid)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int b = blockIdx.x, B = gridDim.x, nch = K >> 3;
  const bf16* xr = x + (long long)b * ldx;
  float ss = 0.f;
  for (int c = threadIdx.x; c < nch; c += 256) {
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c * 8), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += v[j] * v[j];
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float rstd = rsqrtf(tot / (float)K + eps);
  for (int c = threadIdx.x; c < nch; c += 256) {
    float v[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(xr + c * 8), v);
    if (w != nullptr) {
      float wv[8];
      unpack8(*reinterpret_cast<const uint4*>(w + c * 8), wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = wv[j] * bf16r(v[j] * rstd);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = v[j];
    }
    *reinterpret_cast<uint4*>(y + xwin_offset(b, c * 8, B)) = pack8(o);
  }
}

int launch_xwin_norm(const bf16* x, long long ldx, bf16* y, const bf16* w, int B, int K, float eps, cudaStream_t stream) {
  VCL_REQUIRE(K % 8 == 0 && ldx % 8 == 0 && B > 0, "xwin_norm: K=%d / pitch must be x8", K);
  xwin_norm_kernel<<<B, 256, 0, stream>>>(x, ldx, y, w, K, eps);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_fill_int(int* dst, int value, int n, cudaStream_t stream) {
  fill_int_kernel<<<1, 128, 0, stream>>>(dst, value, n);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

int launch_argmax(const float* logits, int* out, long long out_stride, int B, int V,
                  cudaStream_t stream) {
  if (B <= 0) return 0;
  argmax_kernel<<<B, 1024, 0, stream>>>(logits, out, out_stride, V);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

// Decode-time projections: out[b, n] = x[b, :] . W[n, :] for B <= 4 new tokens, CUDA-core version
// over the ROW-MAJOR weights. The default path for 1..4 clips is gemv_tc.cu (bulk-copy ring over a
// slot-ordered weight copy + mma.sync, ~7 % faster); the launch_gemv_* entry points below route
// there when that copy exists and the shape fits, and fall back to this kernel otherwise
// (VCL_GEMV_LEGACY=1, VCL_NO_TILED_WEIGHTS=1, matrices with fewer than 16 rows per SM).
//
// With one token per clip every weight byte is used once per step (13.2 GB per step for the 7B
// model, SURVEY.md section 8d), so these kernels are pure HBM streaming; 5 <= B <= 16 uses
// gemv_mma.cu, larger batches the wgmma GEMM with a narrow N tile.
//
// Work decomposition (one CTA = 16 warps = 512 threads):
//   * the N weight rows are cut into equal contiguous blocks, one per CTA (grid ~ #SMs, so every
//     SM streams the same number of bytes: no tail imbalance);
//   * inside a CTA the K axis is dealt to the 512 lanes in 16-byte chunks (chunk c -> lane c % 512),
//     so a lane needs only J = ceil(K/4096) chunks of the activation vector and keeps them in
//     REGISTERS for the whole kernel (no shared-memory reads in the inner loop);
//   * the CTA walks its rows G at a time: G*J independent 128-bit non-allocating loads per lane are
//     in flight (64 KB per SM), then FMAs, then a warp shuffle reduction per row; the 16 per-warp
//     partials meet in shared memory and the first threads run the epilogue.
//
// Fusions (each removes a launch and an HBM round trip from the 32-layer decode step):
//   prologue  LlamaRMSNorm of x (transformers/models/llama/modeling_llama.py:53-67)
//   epilogue  RES     bf16(bf16(acc) + residual)               (modeling_llama.py:325,331)
//             SWIGLU  silu(gate) * up on interleaved rows      (modeling_llama.py:182-184)
//             QKV     RoPE on q,k + KV-cache append            (modeling_llama.py:124-168,262-270)
//             LOGITS  bf16-rounded logits kept as fp32 for the arg-max
//
// Programmatic dependent launch: the first row group's weight loads are issued BEFORE
// griddepcontrol.wait, so they overlap the tail of the previous kernel in the stream; only the
// activation vector (written by that kernel) is read after the wait.
#include "common.cuh"
#include "kernels.h"

#include <stdlib.h>

namespace vcl {

namespace {

enum { MODE_RES = 0, MODE_SWIGLU = 1, MODE_QKV = 2, MODE_LOGITS = 3 };
constexpr int GEMV_THREADS = 512;
constexpr int GEMV_WARPS = GEMV_THREADS / 32;

struct GemvParams {
  const bf16* x; long long ldx;
  const bf16* W;
  int N, K;
  int rows_per_cta;
  const bf16* norm_w; float eps;
  // RES / SWIGLU
  bf16* out; long long ldo;
  const bf16* res; long long ldr;
  // QKV
  bf16* q_out; long long ldq;
  bf16* kcache; bf16* vcache;
  const bf16* cos_t; const bf16* sin_t;
  int H, s_max, pos;
  const int* pos_dev;
  // LOGITS
  float* logits; long long ldl;
};

__device__ __forceinline__ float silu_bf16(float g) {
  g = bf16r(g);
  return bf16r(__fdividef(g, 1.0f + __expf(-g)));
}

// virtual row v -> weight row. QKV: rows of a RoPE pair (d, d+64) are made adjacent (2p, 2p+1).
template <int MODE>
__device__ __forceinline__ long long map_row(int v) {
  if (MODE == MODE_QKV) {
    const int head_rows = v >> 7;              // (which * H + head)
    const int within = v & 127;
    return (long long)head_rows * 128 + (within >> 1) + ((within & 1) << 6);
  }
  return v;
}

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

__device__ __forceinline__ float dot8(const uint4& w, const uint4& x, float s) {
  s = fmaf(bf16lo(w.x), bf16lo(x.x), s); s = fmaf(bf16hi(w.x), bf16hi(x.x), s);
  s = fmaf(bf16lo(w.y), bf16lo(x.y), s); s = fmaf(bf16hi(w.y), bf16hi(x.y), s);
  s = fmaf(bf16lo(w.z), bf16lo(x.z), s); s = fmaf(bf16hi(w.z), bf16hi(x.z), s);
  s = fmaf(bf16lo(w.w), bf16lo(x.w), s); s = fmaf(bf16hi(w.w), bf16hi(x.w), s);
  return s;
}

template <int NB, int J, int MODE>
__global__ void __launch_bounds__(GEMV_THREADS, (NB * J <= 4) ? 2 : 1) gemv_kernel(const GemvParams p) {
  // rows per group; two groups are kept in flight (software pipeline): 2*G*J 128-bit loads per lane.
  // The register budget is 64/thread so that TWO CTAs fit on an SM: the grid is 2 CTAs per SM, and
  // when a CTA retires the next kernel's CTA (already launched through PDL) starts prefetching
  // its weights in the freed slot while the neighbour is still streaming.
  constexpr int G = (J == 1) ? 4 : (J == 2 ? 2 : 1);
  extern __shared__ __align__(16) float part[];  // [GEMV_WARPS][rows_per_cta][NB]
  __shared__ float red[NB][GEMV_WARPS];
  const int K = p.K;
  const int nch = K >> 3;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.rows_per_cta;
  const int row_begin = blockIdx.x * R;
  const int row_end = min(p.N, row_begin + R);
  const int n_rows = row_end - row_begin;

  auto load_group = [&](int g0, uint4 (&wv)[G][J]) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int r = g0 + g;
      const bf16* wr = p.W + map_row<MODE>(row_begin + (r < n_rows ? r : 0)) * K;
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int c = j * GEMV_THREADS + tid;
        wv[g][j] = (r < n_rows && c < nch) ? ld_nc_v4(wr + c * 8) : make_uint4(0, 0, 0, 0);
      }
    }
  };

  // weights do not depend on the previous kernel: start streaming them before the dependency wait
  uint4 wa[G][J], wb[G][J];
  load_group(0, wa);
  load_group(G, wb);
  pdl_launch_dependents();
  pdl_wait();

  // ---------------- activations: this lane's J chunks per batch row, RMS-normalised ----------------
  uint4 xv[NB][J];
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int c = j * GEMV_THREADS + tid;
      xv[b][j] = (c < nch) ? *reinterpret_cast<const uint4*>(p.x + (long long)b * p.ldx + c * 8)
                           : make_uint4(0, 0, 0, 0);
      if (p.norm_w != nullptr) {
        const uint4 u = xv[b][j];
        const float f0 = bf16lo(u.x), f1 = bf16hi(u.x), f2 = bf16lo(u.y), f3 = bf16hi(u.y);
        const float f4 = bf16lo(u.z), f5 = bf16hi(u.z), f6 = bf16lo(u.w), f7 = bf16hi(u.w);
        ss += f0 * f0 + f1 * f1 + f2 * f2 + f3 * f3 + f4 * f4 + f5 * f5 + f6 * f6 + f7 * f7;
      }
    }
    if (p.norm_w != nullptr) {
      ss = warp_sum(ss);
      if (lane == 0) red[b][warp] = ss;
    }
  }
  if (p.norm_w != nullptr) {
    __syncthreads();
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < GEMV_WARPS; ++w) tot += red[b][w];
      const float rstd = rsqrtf(tot / (float)K + p.eps);
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int c = j * GEMV_THREADS + tid;
        if (c < nch) {
          const uint4 u = xv[b][j];
          const uint4 g = *reinterpret_cast<const uint4*>(p.norm_w + c * 8);
          uint4 o;
          // w * bf16(x * rstd), the product rounded to bf16 again (LlamaRMSNorm)
          o.x = bf16x2_mul(g.x, pack_bf16x2(bf16lo(u.x) * rstd, bf16hi(u.x) * rstd));
          o.y = bf16x2_mul(g.y, pack_bf16x2(bf16lo(u.y) * rstd, bf16hi(u.y) * rstd));
          o.z = bf16x2_mul(g.z, pack_bf16x2(bf16lo(u.z) * rstd, bf16hi(u.z) * rstd));
          o.w = bf16x2_mul(g.w, pack_bf16x2(bf16lo(u.w) * rstd, bf16hi(u.w) * rstd));
          xv[b][j] = o;
        }
      }
    }
  }

  // ---------------- main loop over this CTA's rows: two groups of G rows in flight ----------------
  // single-clip decode: keep the activation chunks unpacked (fp32) so the inner loop only unpacks
  // the weights (8 instead of 16 conversion instructions per 16-byte chunk)
  constexpr bool XF = (NB == 1 && J <= 3);
  float xf[XF ? J : 1][8];
  if (XF) {
#pragma unroll
    for (int j = 0; j < (XF ? J : 1); ++j) {
      const uint4 u = xv[0][j];
      xf[j][0] = bf16lo(u.x); xf[j][1] = bf16hi(u.x); xf[j][2] = bf16lo(u.y); xf[j][3] = bf16hi(u.y);
      xf[j][4] = bf16lo(u.z); xf[j][5] = bf16hi(u.z); xf[j][6] = bf16lo(u.w); xf[j][7] = bf16hi(u.w);
    }
  }
  auto process = [&](int g0, const uint4 (&wv)[G][J]) {
    float acc[G][NB];
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < J; ++j) {
          if (XF) {
            const uint4 w = wv[g][j];
            s = fmaf(bf16lo(w.x), xf[XF ? j : 0][0], s); s = fmaf(bf16hi(w.x), xf[XF ? j : 0][1], s);
            s = fmaf(bf16lo(w.y), xf[XF ? j : 0][2], s); s = fmaf(bf16hi(w.y), xf[XF ? j : 0][3], s);
            s = fmaf(bf16lo(w.z), xf[XF ? j : 0][4], s); s = fmaf(bf16hi(w.z), xf[XF ? j : 0][5], s);
            s = fmaf(bf16lo(w.w), xf[XF ? j : 0][6], s); s = fmaf(bf16hi(w.w), xf[XF ? j : 0][7], s);
          } else {
            s = dot8(wv[g][j], xv[b][j], s);
          }
        }
        acc[g][b] = s;
      }
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float s = warp_sum(acc[g][b]);
        if (lane == 0 && g0 + g < n_rows) part[(warp * R + g0 + g) * NB + b] = s;
      }
  };
  for (int g0 = 0; g0 < n_rows; g0 += 2 * G) {
    process(g0, wa);
    if (g0 + 2 * G < n_rows) load_group(g0 + 2 * G, wa);
    if (g0 + G < n_rows) {
      process(g0 + G, wb);
      if (g0 + 3 * G < n_rows) load_group(g0 + 3 * G, wb);
    }
  }
  __syncthreads();

  // ---------------- epilogue: combine the 16 warp partials ----------------
  constexpr bool PAIRS = (MODE == MODE_SWIGLU || MODE == MODE_QKV);
  const int n_items = (PAIRS ? n_rows / 2 : n_rows) * NB;
  for (int it = tid; it < n_items; it += GEMV_THREADS) {
    const int b = it % NB;
    const int u = it / NB;                         // row (or pair) index inside the CTA block
    const int r0 = PAIRS ? 2 * u : u;
    float v0 = 0.f, v1 = 0.f;
#pragma unroll
    for (int w = 0; w < GEMV_WARPS; ++w) {
      v0 += part[(w * R + r0) * NB + b];
      if (PAIRS) v1 += part[(w * R + r0 + 1) * NB + b];
    }
    const int vrow = row_begin + r0;               // virtual row
    if (MODE == MODE_RES) {
      float y = bf16r(v0);
      if (p.res != nullptr) y += __bfloat162float(p.res[(long long)b * p.ldr + vrow]);
      p.out[(long long)b * p.ldo + vrow] = __float2bfloat16_rn(y);
    } else if (MODE == MODE_LOGITS) {
      p.logits[(long long)b * p.ldl + vrow] = bf16r(v0);
    } else if (MODE == MODE_SWIGLU) {
      p.out[(long long)b * p.ldo + (vrow >> 1)] = __float2bfloat16_rn(silu_bf16(v0) * bf16r(v1));
    } else {  // MODE_QKV: vrow = (which*H + head)*128 + 2*d
      const int hr = vrow >> 7;
      const int which = hr / p.H, head = hr - which * p.H;
      const int d = (vrow & 127) >> 1;
      const float lo = bf16r(v0), hi = bf16r(v1);
      const int pos = p.pos + (p.pos_dev != nullptr ? __ldg(p.pos_dev) : 0);
      const long long coff = (((long long)b * p.H + head) * p.s_max + pos) * 128;
      if (which == 2) {
        p.vcache[coff + d] = __float2bfloat16_rn(lo);
        p.vcache[coff + d + 64] = __float2bfloat16_rn(hi);
      } else {
        const float c = __bfloat162float(p.cos_t[(long long)pos * 64 + d]);
        const float s = __bfloat162float(p.sin_t[(long long)pos * 64 + d]);
        const float olo = bf16r(lo * c) + bf16r(-hi * s);
        const float ohi = bf16r(hi * c) + bf16r(lo * s);
        if (which == 0) {
          p.q_out[(long long)b * p.ldq + head * 128 + d] = __float2bfloat16_rn(olo);
          p.q_out[(long long)b * p.ldq + head * 128 + d + 64] = __float2bfloat16_rn(ohi);
        } else {
          p.kcache[coff + d] = __float2bfloat16_rn(olo);
          p.kcache[coff + d + 64] = __float2bfloat16_rn(ohi);
        }
      }
    }
  }
}

template <int NB, int J, int MODE>
int launch_j(GemvParams p, cudaStream_t stream) {
  // CTAs per SM in the grid (two fit: 64 registers per thread). VCL_GEMV_CTAS_PER_SM=1 leaves the
  // second slot to the NEXT kernel's CTAs, which PDL lets start prefetching weights early.
  static const int per_sm = getenv("VCL_GEMV_CTAS_PER_SM") ? atoi(getenv("VCL_GEMV_CTAS_PER_SM")) : 2;
  // batches whose activation registers do not fit the 64-register budget run one CTA per SM
  int grid = ((NB * J <= 4) ? (per_sm > 0 ? per_sm : 2) : 1) * device_num_sms();
  int R = (p.N + grid - 1) / grid;
  if (R & 1) ++R;                                   // pair modes need whole pairs per CTA
  if (R < 2) R = 2;
  grid = (p.N + R - 1) / R;
  p.rows_per_cta = R;
  const size_t smem = (size_t)GEMV_WARPS * R * NB * sizeof(float);
  VCL_REQUIRE(smem <= 100 * 1024, "gemv: %d rows per CTA need %zu bytes of shared memory", R, smem);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(GEMV_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, gemv_kernel<NB, J, MODE>, p));
  count_launches(1);
  return 0;
}

template <int NB, int MODE>
int launch_nb(const GemvParams& p, cudaStream_t stream) {
  const int J = (p.K / 8 + GEMV_THREADS - 1) / GEMV_THREADS;
  switch (J) {
    case 1: return launch_j<NB, 1, MODE>(p, stream);
    case 2: return launch_j<NB, 2, MODE>(p, stream);
    case 3: return launch_j<NB, 3, MODE>(p, stream);
    case 4: return launch_j<NB, 4, MODE>(p, stream);
  }
  set_last_error("gemv: K=%d too large (max 16384)", p.K);
  return -1;
}

template <int MODE>
int launch_mode(int B, const GemvParams& p, cudaStream_t stream) {
  VCL_REQUIRE(B >= 1 && B <= 4, "gemv: batch %d outside 1..4 (larger batches use the wgmma GEMM)", B);
  VCL_REQUIRE(p.K % 8 == 0 && p.ldx % 8 == 0, "gemv: K and pitch must be multiples of 8");
  VCL_REQUIRE(((uintptr_t)p.x % 16) == 0 && ((uintptr_t)p.W % 16) == 0, "gemv: 16-byte alignment required");
  switch (B) {
    case 1: return launch_nb<1, MODE>(p, stream);
    case 2: return launch_nb<2, MODE>(p, stream);
    case 3: return launch_nb<3, MODE>(p, stream);
    default: return launch_nb<4, MODE>(p, stream);
  }
}

template <int NB, int MODE>
int init_nb() {
  const int cap = 100 * 1024;
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_kernel<NB, 1, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_kernel<NB, 2, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_kernel<NB, 3, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_kernel<NB, 4, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap));
  return 0;
}

template <int MODE>
int init_mode() {
  if (init_nb<1, MODE>() || init_nb<2, MODE>() || init_nb<3, MODE>() || init_nb<4, MODE>()) return -2;
  return 0;
}

GemvParams base_params(const GemvArgs& g) {
  GemvParams p = {};
  p.x = g.x; p.ldx = g.ldx; p.W = g.W; p.N = g.N; p.K = g.K;
  p.norm_w = g.norm_w; p.eps = g.eps;
  return p;
}

}  // namespace

int init_gemv_kernels() {
  if (init_mode<MODE_RES>() || init_mode<MODE_SWIGLU>() || init_mode<MODE_QKV>() ||
      init_mode<MODE_LOGITS>()) return -2;
  return 0;
}

int launch_gemv_residual(const GemvArgs& g, bf16* out, long long ldo, const bf16* res,
                         long long ldr, cudaStream_t stream) {
  if (gemv_tc_supported(g)) return launch_gemv_tc_residual(g, out, ldo, res, ldr, stream);
  GemvParams p = base_params(g);
  p.out = out; p.ldo = ldo; p.res = res; p.ldr = ldr;
  return launch_mode<MODE_RES>(g.B, p, stream);
}

int launch_gemv_swiglu(const GemvArgs& g, bf16* out, long long ldo, cudaStream_t stream) {
  VCL_REQUIRE(g.N % 2 == 0, "gemv swiglu: N must be even (interleaved gate/up rows)");
  if (gemv_tc_supported(g)) return launch_gemv_tc_swiglu(g, out, ldo, stream);
  GemvParams p = base_params(g);
  p.out = out; p.ldo = ldo;
  return launch_mode<MODE_SWIGLU>(g.B, p, stream);
}

int launch_gemv_qkv_rope(const GemvArgs& g, bf16* q_out, long long ldq, bf16* kcache, bf16* vcache,
                         const bf16* cos_t, const bf16* sin_t, int H, int head_dim, int s_max,
                         int pos, cudaStream_t stream, const int* pos_dev) {
  VCL_REQUIRE(head_dim == 128, "gemv qkv: head_dim must be 128");
  VCL_REQUIRE(g.N == 3 * H * 128, "gemv qkv: N=%d != 3*H*128", g.N);
  VCL_REQUIRE(pos >= 0 && pos < s_max, "gemv qkv: position %d outside the cache (%d)", pos, s_max);
  if (gemv_tc_supported(g))
    return launch_gemv_tc_qkv_rope(g, q_out, ldq, kcache, vcache, cos_t, sin_t, H, s_max, pos, stream, pos_dev);
  VCL_REQUIRE(g.embed == nullptr, "gemv qkv: the fused embedding gather needs the ring kernel (gemv_tc)");
  GemvParams p = base_params(g);
  p.q_out = q_out; p.ldq = ldq; p.kcache = kcache; p.vcache = vcache;
  p.cos_t = cos_t; p.sin_t = sin_t; p.H = H; p.s_max = s_max; p.pos = pos; p.pos_dev = pos_dev;
  return launch_mode<MODE_QKV>(g.B, p, stream);
}

int launch_gemv_logits(const GemvArgs& g, float* logits, long long ldl, cudaStream_t stream) {
  if (gemv_tc_supported(g)) return launch_gemv_tc_logits(g, logits, ldl, stream);
  GemvParams p = base_params(g);
  p.logits = logits; p.ldl = ldl;
  return launch_mode<MODE_LOGITS>(g.B, p, stream);
}

}  // namespace vcl

// Decode projections for 5..16 clips per GPU: out[b][n] = x[b] . W[n, :], weights streamed ONCE.
//
// Same streaming machinery as gemv_tc.cu (the 1..4-clip kernel): one CTA per SM, a producer warp that
// fills a shared-memory ring with one cp.async.bulk per 16 KB slot of the slot-ordered weight copy
// (gemv_tc_repack: [16-row group][512-k chunk] blocks already in mma.sync A-fragment order), weights
// requested BEFORE the dependency wait, all 8 consumer warps working on every slot (each takes every
// eighth 32-wide K block), so a slot is free again ~100 cycles after it landed and almost the whole ring
// is in flight from HBM at any time. What changes with up to 16 activation vectors:
//
//   * they no longer fit in shared memory next to the ring (16 x 11008 x 2 B = 352 KB for down_proj), so
//     the K dimension is walked chunk-major: for every 512-wide K chunk the producer first copies that
//     WINDOW of the (already normalised) activations and then the slots of that chunk for all row groups
//     of the CTA. The slots are contiguous 16 KB blocks whatever the order they are visited in, so the
//     same weight copy serves both kernels. The activations are kept in global memory window-major
//     ("xwin": element (b, k) at ((k / 512) * B + b) * 544 + k % 512), so that a window is ONE contiguous
//     bulk copy -- the copy engine retires ~23 copies per microsecond and SM whatever their size, sixteen
//     1 KB row copies per chunk made o_proj / down_proj copy-rate bound -- and its rows arrive already
//     padded to 1088 B, which makes the B-fragment loads of the 8 clips of an MMA bank-conflict free.
//     Whoever produces an input of this kernel writes that layout: the decode-path RMSNorm
//     (launch_xwin_norm), the decode attention kernel and this kernel's own SwiGLU epilogue.
//   * the accumulators of ALL row groups of the CTA (up to 14 groups x 2 MMA column blocks x 4 registers
//     per warp) stay in registers across the K chunks; the 8 per-warp partial tiles of a group meet once,
//     at the end, in the (then idle) ring memory.
//   * clip b is column b of the m16n8k16 B operand: two column blocks cover 16 clips.
//
// A warp per row group (no reduction at all) keeps a slot held for ~1000 cycles by its one consumer, so only
// a few of the ring slots are in flight; per-row window copies make the copy engine the limit.
//
// Epilogues (RoPE + KV append, SwiGLU, residual, logits) and every rounding point are those of
// gemv_tc.cu / gemv.cu (reference: transformers/models/llama/modeling_llama.py:124-168 RoPE, :171-184
// MLP, :325,331 residuals).
#include "common.cuh"
#include "kernels.h"

#include <stdlib.h>

namespace vcl {

namespace {

constexpr int TW_CWARPS = 8;
constexpr int TW_THREADS = TW_CWARPS * 32 + 32;
constexpr int TW_KC = 512;
constexpr int TW_SLOT_BYTES = 16 * TW_KC * 2;          // 16 KB
constexpr int TW_SLOTS = 8;                            // power of two; 128 KB, re-used by the final reduction
constexpr int TW_XROW = XWIN_PITCH * 2;                // 1088 bytes per activation row of a window
constexpr int TW_XBUF = 16 * TW_XROW;                  // one window of 16 clips
constexpr int TW_XWIN = 4;                             // activation windows in flight (power of two): with two, a
                                                       // CTA that owns 1-2 row groups (o_proj, down_proj) waited
                                                       // an L2 round trip for a window every second chunk
constexpr int TW_SMEM = TW_SLOTS * TW_SLOT_BYTES + TW_XWIN * TW_XBUF + 256;
constexpr int TW_TILE = 16 * 17;                       // floats of one partial tile (16 rows x 16 clips, padded rows)

enum { TW_RES = 0, TW_SWIGLU = 1, TW_QKV = 2, TW_LOGITS = 3 };

struct TwParams {
  int mode;
  const bf16* W_tiled; int N, K;
  const bf16* x; int B;               // activations in xwin layout
  bf16* out; long long ldo; int out_xwin;   // out_xwin: SwiGLU output written in xwin layout (feeds down_proj)
  const bf16* res; long long ldr;
  bf16* q_out; long long ldq;
  bf16* kcache; bf16* vcache;
  float* logits; long long ldl;
  const bf16* cos_t; const bf16* sin_t;
  int H, s_max, pos;
  const int* pos_dev;
};

__device__ __forceinline__ void tw_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tw_mma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                       uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void tw_cbar() {            // barrier among the consumer warps only
  asm volatile("bar.sync 1, %0;" ::"r"(TW_CWARPS * 32) : "memory");
}

// NG = upper bound of the row groups a CTA owns (the accumulator arrays are sized and unrolled by it)
template <int NG>
__global__ void __launch_bounds__(TW_THREADS, 1) gemv_tcw_kernel(const TwParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  // layout: ring[8] (after the main loop: partial tiles [warp][group]) | x windows [4][16][1088 B] | barriers
  uint8_t* xs = smem + TW_SLOTS * TW_SLOT_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(xs + TW_XWIN * TW_XBUF);
  const uint32_t ring0 = smem_u32(smem), xs0 = smem_u32(xs), bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (TW_SLOTS + s); };
  auto xfull_bar = [&](int s) { return bar0 + 8u * (2 * TW_SLOTS + s); };
  auto xempty_bar = [&](int s) { return bar0 + 8u * (2 * TW_SLOTS + TW_XWIN + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = p.K, N = p.N, NB = p.B;
  const int nkc = (K + TW_KC - 1) / TW_KC;
  const int n_groups = (N + 15) >> 4;
  const int grp_begin = (int)(((long long)blockIdx.x * n_groups) / gridDim.x);
  const int ng = (int)(((long long)(blockIdx.x + 1) * n_groups) / gridDim.x) - grp_begin;   // 1..NG

  if (tid == 0) {
    for (int s = 0; s < TW_SLOTS; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), TW_CWARPS); }
    for (int s = 0; s < TW_XWIN; ++s) { mbar_init(xfull_bar(s), 1); mbar_init(xempty_bar(s), TW_CWARPS); }
    mbar_fence_init();
  }
  // rows of the activation windows that no clip owns stay zero (their MMA columns are never stored)
  for (int i = tid; i < TW_XWIN * TW_XBUF / 16; i += TW_THREADS) reinterpret_cast<uint4*>(xs)[i] = make_uint4(0, 0, 0, 0);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp == TW_CWARPS) {
    // =============================== producer ===============================
    // (32-bit index arithmetic only: a 64-bit division here becomes a subroutine call inside the
    // single-lane region and the uniform-datapath code around the bulk copies then faults)
    if (lane == 0) {
      const int total = ng * nkc;
      const int pre = total < TW_SLOTS ? total : TW_SLOTS;
      // the weights never depend on the previous kernel: fill the ring before the dependency wait
      {
        int kc = 0, lg = 0;
        for (int idx = 0; idx < pre; ++idx) {
          const uint32_t bytes = (uint32_t)min(TW_KC, K - kc * TW_KC) * 32u;
          const bf16* src = p.W_tiled + (size_t)(grp_begin + lg) * 16 * K + (size_t)kc * TW_KC * 16;
          mbar_arrive_expect_tx(full_bar(idx), bytes);
          tw_bulk_g2s(ring0 + idx * TW_SLOT_BYTES, src, bytes, full_bar(idx));
          if (++lg == ng) { lg = 0; ++kc; }
        }
      }
      asm volatile("griddepcontrol.wait;" ::: "memory");
      int idx = 0, slot = 0, use = 0;                 // slot = idx % TW_SLOTS, use = idx / TW_SLOTS
      const uint32_t win_bytes = (uint32_t)NB * TW_XROW;
      for (int kc = 0; kc < nkc; ++kc) {
        const int xb = kc & (TW_XWIN - 1);
        if (kc >= TW_XWIN) mbar_wait(xempty_bar(xb), (uint32_t)(((kc / TW_XWIN) - 1) & 1));
        mbar_arrive_expect_tx(xfull_bar(xb), win_bytes);
        tw_bulk_g2s(xs0 + xb * TW_XBUF, p.x + (size_t)kc * NB * XWIN_PITCH, win_bytes, xfull_bar(xb));
        for (int lg = 0; lg < ng; ++lg) {
          if (idx >= pre) {
            const uint32_t bytes = (uint32_t)min(TW_KC, K - kc * TW_KC) * 32u;
            const bf16* src = p.W_tiled + (size_t)(grp_begin + lg) * 16 * K + (size_t)kc * TW_KC * 16;
            mbar_wait(empty_bar(slot), (uint32_t)((use - 1) & 1));
            mbar_arrive_expect_tx(full_bar(slot), bytes);
            tw_bulk_g2s(ring0 + slot * TW_SLOT_BYTES, src, bytes, full_bar(slot));
          }
          ++idx;
          if (++slot == TW_SLOTS) { slot = 0; ++use; }
        }
      }
    }
    return;
  }

  // =============================== consumers ===============================
  asm volatile("griddepcontrol.wait;" ::: "memory");   // the epilogue reads / overwrites tensors of earlier kernels
  const int g = lane >> 2, q = lane & 3;
  float acc[NG][2][4];
#pragma unroll
  for (int a = 0; a < NG; ++a)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[a][j][e] = 0.f;

  int slot = 0;
  uint32_t par = 0;
  for (int kc = 0; kc < nkc; ++kc) {
    const int xb = kc & (TW_XWIN - 1);
    const int kb_n = min(TW_KC, K - kc * TW_KC) >> 5;       // 32-wide K blocks in this chunk
    mbar_wait(xfull_bar(xb), (uint32_t)((kc / TW_XWIN) & 1));
    const uint8_t* xw = xs + xb * TW_XBUF;
    // this warp's share of every slot of the chunk: K blocks warp and warp + 8; the B fragments (the
    // activations of 16 clips for those K blocks) are the same for every row group: load them once
    uint4 xq[2][2];
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
      for (int j = 0; j < 2; ++j)
        xq[t][j] = *reinterpret_cast<const uint4*>(xw + (8 * j + g) * TW_XROW + (warp + TW_CWARPS * t) * 64 + q * 16);   // clip 8j+g
#pragma unroll
    for (int a = 0; a < NG; ++a) {
      if (a < ng) {
        mbar_wait(full_bar(slot), par);
        const uint8_t* base = smem + slot * TW_SLOT_BYTES;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int kb = warp + TW_CWARPS * t;
          if (kb < kb_n) {
            const uint4 wa = *reinterpret_cast<const uint4*>(base + kb * 1024 + lane * 16);          // row g
            const uint4 wb = *reinterpret_cast<const uint4*>(base + kb * 1024 + 512 + lane * 16);    // row g + 8
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              tw_mma(acc[a][j], wa.x, wb.x, wa.y, wb.y, xq[t][j].x, xq[t][j].y);
              tw_mma(acc[a][j], wa.z, wb.z, wa.w, wb.w, xq[t][j].z, xq[t][j].w);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(slot));
        if (++slot == TW_SLOTS) { slot = 0; par ^= 1u; }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(xempty_bar(xb));
  }

  // ---------------- the 8 per-warp partial tiles of every group meet in the (now idle) ring ----------------
  tw_cbar();                                            // every warp has left the ring
  float* tiles = reinterpret_cast<float*>(smem);        // [warp][group][16][17]
#pragma unroll
  for (int a = 0; a < NG; ++a) {
    if (a < ng) {
      float* t = tiles + ((size_t)warp * NG + a) * TW_TILE;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        t[g * 17 + 8 * j + 2 * q] = acc[a][j][0];
        t[g * 17 + 8 * j + 2 * q + 1] = acc[a][j][1];
        t[(g + 8) * 17 + 8 * j + 2 * q] = acc[a][j][2];
        t[(g + 8) * 17 + 8 * j + 2 * q + 1] = acc[a][j][3];
      }
    }
  }
  tw_cbar();

  // ---------------- fused epilogue ----------------
  // All 256 consumer threads share the items of every group: thread = (row or row pair, clip) with the ROW
  // index fastest, so that a warp's accesses to the residual / output rows are contiguous runs (a warp per
  // group walking (row, clip) items with the clip fastest touched 32 sectors per instruction, one dependent
  // round trip per 32 items at the end of every launch). The 8 partial tiles are summed on the fly,
  // in a fixed order.
  const int mode = p.mode;
  const bool pairs = (mode == TW_SWIGLU || mode == TW_QKV);
  const int pos = p.pos + (p.pos_dev != nullptr ? __ldg(p.pos_dev) : 0);
  auto tile_sum = [&](int lg, int e) {
    float v = tiles[(size_t)lg * TW_TILE + e];
#pragma unroll
    for (int w2 = 1; w2 < TW_CWARPS; ++w2) v += tiles[((size_t)w2 * NG + lg) * TW_TILE + e];
    return v;
  };
  if (!pairs) {
    const int rr = tid & 15, b = tid >> 4;               // 16 rows x 16 clips of one group per pass
#pragma unroll 2
    for (int lg = 0; lg < ng; ++lg) {
      const int vrow = (grp_begin + lg) * 16 + rr;
      if (b < NB && vrow < N) {
        const float v0 = tile_sum(lg, rr * 17 + b);
        if (mode == TW_RES) {
          float y = bf16r(v0);
          if (p.res != nullptr) y += __bfloat162float(p.res[(long long)b * p.ldr + vrow]);
          p.out[(long long)b * p.ldo + vrow] = __float2bfloat16_rn(y);
        } else {
          p.logits[(long long)b * p.ldl + vrow] = bf16r(v0);
        }
      }
    }
  } else {
    const int pr = tid & 7, b = (tid >> 3) & 15;         // 8 row pairs x 16 clips of TWO groups per pass
    for (int lg = tid >> 7; lg < ng; lg += 2) {
      const int rr = 2 * pr;
      const int vrow = (grp_begin + lg) * 16 + rr;
      if (b >= NB || vrow >= N) continue;
      const float v0 = tile_sum(lg, rr * 17 + b), v1 = tile_sum(lg, (rr + 1) * 17 + b);
      if (mode == TW_SWIGLU) {
        const float gt = bf16r(v0);
        const float sg = bf16r(__fdividef(gt, 1.0f + __expf(-gt)));
        const int col = vrow >> 1;
        const long long o = p.out_xwin ? (long long)xwin_offset(b, col, NB) : (long long)b * p.ldo + col;
        p.out[o] = __float2bfloat16_rn(sg * bf16r(v1));
      } else {  // TW_QKV: vrow = (which*H + head)*128 + 2*d
        const int hr = vrow >> 7;
        const int which = hr / p.H, head = hr - which * p.H;
        const int d = (vrow & 127) >> 1;
        const float lo = bf16r(v0), hi = bf16r(v1);
        const long long coff = (((long long)b * p.H + head) * p.s_max + pos) * 128;
        if (which == 2) {
          p.vcache[coff + d] = __float2bfloat16_rn(lo);
          p.vcache[coff + d + 64] = __float2bfloat16_rn(hi);
        } else {
          const float cs = __bfloat162float(p.cos_t[(long long)pos * 64 + d]);
          const float sn = __bfloat162float(p.sin_t[(long long)pos * 64 + d]);
          const float olo = bf16r(lo * cs) + bf16r(-hi * sn);
          const float ohi = bf16r(hi * cs) + bf16r(lo * sn);
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
}

TwParams tw_base(const GemvArgs& g, int mode) {
  TwParams p = {};
  p.mode = mode; p.W_tiled = g.W_tiled; p.N = g.N; p.K = g.K; p.x = g.x; p.B = g.B;
  return p;
}

int tw_launch(const TwParams& p, cudaStream_t stream) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(device_num_sms());
  cfg.blockDim = dim3(TW_THREADS);
  cfg.dynamicSmemBytes = TW_SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const int ng_max = ((p.N + 15) / 16 + (int)cfg.gridDim.x - 1) / (int)cfg.gridDim.x;     // groups of the busiest CTA
  if (ng_max <= 2) VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, gemv_tcw_kernel<2>, p));
  else if (ng_max <= 6) VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, gemv_tcw_kernel<6>, p));
  else if (ng_max <= 10) VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, gemv_tcw_kernel<10>, p));
  else VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, gemv_tcw_kernel<14>, p));
  count_launches(1);
  return 0;
}

}  // namespace

int init_gemv_tcw_kernels() {
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_tcw_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, TW_SMEM));
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_tcw_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, TW_SMEM));
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_tcw_kernel<10>, cudaFuncAttributeMaxDynamicSharedMemorySize, TW_SMEM));
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_tcw_kernel<14>, cudaFuncAttributeMaxDynamicSharedMemorySize, TW_SMEM));
  return 0;
}

// 5..16 clips, a slot-ordered weight copy, between 1 and 14 row groups per CTA; g.x is in xwin layout
bool gemv_tcw_supported(const GemvArgs& g) {
  static const bool off = getenv("VCL_GEMV_TCW_OFF") != nullptr;   // A/B switch: fall back to gemv_mma
  if (off || g.W_tiled == nullptr || g.norm_w != nullptr || g.B < 5 || g.B > 16) return false;
  if (g.K % 32 != 0 || ((uintptr_t)g.x % 16) != 0 || ((uintptr_t)g.W_tiled % 16) != 0) return false;
  const int n_groups = (g.N + 15) / 16, grid = device_num_sms();
  return n_groups >= grid && n_groups <= 14 * grid;
}

int launch_gemv_tcw_residual(const GemvArgs& g, bf16* out, long long ldo, const bf16* res, long long ldr,
                             cudaStream_t stream) {
  VCL_REQUIRE(gemv_tcw_supported(g), "gemv_tcw: unsupported problem B=%d N=%d K=%d", g.B, g.N, g.K);
  TwParams p = tw_base(g, TW_RES);
  p.out = out; p.ldo = ldo; p.res = res; p.ldr = ldr;
  return tw_launch(p, stream);
}

int launch_gemv_tcw_swiglu(const GemvArgs& g, bf16* out, long long ldo, bool out_xwin, cudaStream_t stream) {
  VCL_REQUIRE(gemv_tcw_supported(g) && g.N % 2 == 0, "gemv_tcw swiglu: unsupported problem B=%d N=%d K=%d", g.B, g.N, g.K);
  TwParams p = tw_base(g, TW_SWIGLU);
  p.out = out; p.ldo = ldo; p.out_xwin = out_xwin ? 1 : 0;
  return tw_launch(p, stream);
}

int launch_gemv_tcw_qkv_rope(const GemvArgs& g, bf16* q_out, long long ldq, bf16* kcache, bf16* vcache,
                             const bf16* cos_t, const bf16* sin_t, int H, int s_max, int pos, cudaStream_t stream,
                             const int* pos_dev) {
  VCL_REQUIRE(gemv_tcw_supported(g) && g.N == 3 * H * 128, "gemv_tcw qkv: unsupported problem B=%d N=%d K=%d", g.B, g.N, g.K);
  TwParams p = tw_base(g, TW_QKV);
  p.q_out = q_out; p.ldq = ldq; p.kcache = kcache; p.vcache = vcache;
  p.cos_t = cos_t; p.sin_t = sin_t; p.H = H; p.s_max = s_max; p.pos = pos; p.pos_dev = pos_dev;
  return tw_launch(p, stream);
}

int launch_gemv_tcw_logits(const GemvArgs& g, float* logits, long long ldl, cudaStream_t stream) {
  VCL_REQUIRE(gemv_tcw_supported(g), "gemv_tcw logits: unsupported problem B=%d N=%d K=%d", g.B, g.N, g.K);
  TwParams p = tw_base(g, TW_LOGITS);
  p.logits = logits; p.ldl = ldl;
  return tw_launch(p, stream);
}

}  // namespace vcl

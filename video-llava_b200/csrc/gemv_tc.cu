// Decode projections for 1..4 clips: out[b][n] = x[b] . W[n, :], one kernel per weight matrix.
//
// What bounds these kernels is how much of the time HBM is kept streaming:
//   * a chain of per-matrix kernels keeps HBM busier with programmatic dependent launch (the next
//     kernel's first loads are in flight while the current one drains) than when every kernel starts cold;
//   * cp.async.bulk rings cost no registers and no issue slots in the consumer warps, but the copy engine
//     retires a limited number of copies per SM whatever their size, so the slots have to be contiguous
//     in memory and fetched with ONE copy each;
//   * mma.sync does the K reduction in the tensor pipe at a few instructions per KB of weights, where a
//     CUDA-core GEMV spends tens (unpack, FMA, warp shuffle reduction);
//   * the serial latency after griddepcontrol.wait (activation fetch + norm) is dead time for HBM
//     once the ring is full, so it is kept to one L2 round trip.
//
// Structure (one CTA per SM, at most one per 16-row group; 9 warps, 8 x 16 KB ring):
//   warp 8      producer: walks this CTA's 16-row groups, K chunk by K chunk (512 k), and fills
//               the ring with one bulk copy per slot. The kernel reads a decode-only copy of the
//               matrix that the weight loader lays out slot by slot (gemv_tc_repack below):
//               [16-row group][K chunk][32-wide K block][row half][lane] x 16 bytes, i.e. already
//               in mma.sync A-fragment order. Weights never depend on the previous kernel, so
//               the producer starts immediately, BEFORE the dependency wait.
//   warps 0-7   consumers: griddepcontrol.wait, stage the activation vector in shared memory (bf16,
//               optionally RMS-normalised), then per slot two m16n8k16 MMAs per 32-wide K block:
//               A fragments with two conflict-free LDS.128 (lane l reads bytes [16 l, 16 l + 16)
//               of each 512-byte row half), column 0 of the B fragment from the activation
//               vector. fp32 accumulators live across the K chunks of a row group; the 8 per-warp
//               partials meet in shared memory after every group and the fused epilogues (RoPE +
//               KV append, SwiGLU, residual, logits) run once at the end.
// Ring depth: 8 slots by default (VCL_GEMV_TC_SLOTS overrides it for A/B runs); not re-tuned on the H100.
//
// Rounding points (reference: transformers/models/llama/modeling_llama.py:53-67 RMSNorm, :124-168 RoPE,
// :171-184 MLP, :325,331 residuals): the normalised activation w * bf16(x * rstd) is rounded to bf16, every
// projection is rounded to bf16 before its epilogue, and so are the RoPE products, silu(gate) and the
// residual sum; logits are kept bf16-rounded in fp32.
#include "common.cuh"
#include "kernels.h"

#include <stdio.h>
#include <stdlib.h>

#include <vector>

namespace vcl {

namespace {

constexpr int TC_CWARPS = 8;
constexpr int TC_CONSUMERS = TC_CWARPS * 32;
constexpr int TC_THREADS = TC_CONSUMERS + 32;
constexpr int TC_KC = 512;                          // k elements per slot
constexpr int TC_SLOT_BYTES = 16 * TC_KC * 2;       // 16 KB, one bulk copy
constexpr int TC_MAX_SLOTS = 14;                    // barrier array size
constexpr int TC_DEFAULT_SLOTS = 8;
constexpr int TC_SMEM_BUDGET = 160 * 1024;          // one CTA per SM; the rest of the SM stays free for the
                                                    // attention kernel's CTAs, which launch early (PDL)

enum { TC_MODE_RES = 0, TC_MODE_SWIGLU = 1, TC_MODE_QKV = 2, TC_MODE_LOGITS = 3 };

struct TcParams {
  GemvArgs a;                       // the projection; a.B clips (1..4) are the columns of the MMA B operand
  int mode;
  bf16* out; long long ldo;         // RES: out[B][N] (+res); SWIGLU: out[B][N/2]
  const bf16* res; long long ldr;
  bf16* q_out; long long ldq;       // QKV: q [B][ldq], cache base of the layer [B][H][S][128]
  bf16* kcache; bf16* vcache;
  const bf16* cos_t; const bf16* sin_t;
  int H, s_max, pos;
  const int* pos_dev;               // position = pos + *pos_dev (one captured graph for every prompt length)
  float* logits; long long ldl;     // LOGITS: [B][ldl] bf16-rounded fp32 (null: not stored)
  int n_slots;
  int x_elems;                      // activation buffer (elements)
  int r_cap;                        // rows one CTA owns at most (result buffer)
  unsigned long long* trace;        // optional [grid][8] timestamps (VCL_TC_TRACE)
};

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
__device__ __forceinline__ uint4 ld_cg_v4(const void* p) {     // served by L2: never a stale L1 line
  uint4 r;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void cbar() {            // barrier among the consumer warps only
  asm volatile("bar.sync 1, %0;" ::"r"(TC_CONSUMERS) : "memory");
}
__device__ __forceinline__ void tc_mma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                       uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// virtual q/k/v row -> weight row: the rows of a RoPE pair (d, d+64) are made adjacent (2p, 2p+1)
__device__ __forceinline__ long long qkv_row(int v) {
  return (long long)(v >> 7) * 128 + ((v & 127) >> 1) + (((v & 127) & 1) << 6);
}

__global__ void __launch_bounds__(TC_THREADS, 2) gemv_tc_kernel(const TcParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  // layout: ring[n_slots] | x[nb][K] bf16 | pbuf[2][TC_CWARPS][16][4] | result[r_cap][4] fp32 | red | barriers
  const int n_slots = p.n_slots;
  bf16* xs = reinterpret_cast<bf16*>(smem + (size_t)n_slots * TC_SLOT_BYTES);
  float* pbuf = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(xs) + (size_t)p.x_elems * 2);
  float* result = pbuf + 2 * TC_CWARPS * 16 * 4;
  float* red = result + p.r_cap * 4;
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + 4 * TC_CWARPS);
  const uint32_t ring0 = smem_u32(smem);
  const uint32_t bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (TC_MAX_SLOTS + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  auto trace = [&](int ev) {
    if (p.trace != nullptr) p.trace[(size_t)blockIdx.x * 8 + ev] = globaltimer_ns();
  };
  if (tid == 0) {
    trace(0);
    for (int s = 0; s < n_slots; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), TC_CWARPS); }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();                           // the next kernel (attention) may become resident

  const GemvArgs& a = p.a;
  int slot = 0;
  uint32_t par = 0;
  auto advance = [&]() { if (++slot == n_slots) { slot = 0; par ^= 1u; } };
  // contiguous blocks of 16-row groups per CTA, sizes differing by at most one group, the larger shares
  // spread evenly over the grid
  auto my_groups = [&](int N, int& grp_begin) {
    const int n_groups = (N + 15) >> 4;
    grp_begin = (int)(((long long)blockIdx.x * n_groups) / gridDim.x);
    return (int)(((long long)(blockIdx.x + 1) * n_groups) / gridDim.x) - grp_begin;
  };

  if (warp == TC_CWARPS) {
    // =============================== producer ===============================
    // never waits for the consumers' epilogue or activation fetch: HBM keeps streaming meanwhile
    if (lane == 0) {
      const int K = a.K, nkc = (K + TC_KC - 1) / TC_KC;
      int grp_begin;
      const int ng = my_groups(a.N, grp_begin);
      trace(5);
      for (int g = 0; g < ng; ++g) {
        const bf16* src = a.W_tiled + (size_t)(grp_begin + g) * 16 * K;
        for (int kc = 0; kc < nkc; ++kc) {
          const uint32_t bytes = (uint32_t)min(TC_KC, K - kc * TC_KC) * 32u;    // 16 rows x 2 B
          mbar_wait(empty_bar(slot), par ^ 1u);
          mbar_arrive_expect_tx(full_bar(slot), bytes);
          bulk_g2s(ring0 + slot * TC_SLOT_BYTES, src + (size_t)kc * TC_KC * 16, bytes, full_bar(slot));
          advance();
        }
      }
      trace(6);
    }
    return;
  }

  // =============================== consumers ===============================
  constexpr int XU = 7;                               // 16-byte chunks per thread: K <= 14336
  const int g = lane >> 2, q = lane & 3;
  const int K = a.K, N = a.N, mode = p.mode;
  const int nkc = (K + TC_KC - 1) / TC_KC;
  const int nch = K >> 3;
  int grp_begin;
  const int ng = my_groups(N, grp_begin);
  const int row0 = grp_begin * 16;
  // Activation vector -> shared memory (bf16), RMS-normalised when the layer norm is fused. The
  // norm weights (constants) are parked in the x buffer first, every thread issues its x loads back
  // to back: the dependent latency is one L2 round trip.
  const int NB = a.B;
  if (NB > 1) {
    // ---- 2-4 clips: every clip's vector is fetched at once (cp.async.cg straight into the x buffer:
    // ONE L2 round trip for the launch instead of one per clip), then normalised in place. The norm
    // weights (constants, the same for every clip) are parked behind the x buffer before the dependency wait.
    bf16* nw = xs + (size_t)NB * K;                 // the plan reserves K more elements for launches with a norm
    if (a.norm_w != nullptr) {
#pragma unroll
      for (int u = 0; u < XU; ++u) {
        const int c = tid + u * TC_CONSUMERS;
        if (c < nch) *reinterpret_cast<uint4*>(nw + c * 8) = __ldg(reinterpret_cast<const uint4*>(a.norm_w + c * 8));
      }
    }
    pdl_wait();
    if (tid == 0) trace(1);
    const bf16* xg[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) xg[b] = a.x + (long long)(b < NB ? b : 0) * a.ldx;
    if (a.embed != nullptr) {
      int tok[4] = {0, 0, 0, 0};
      if (a.amax_in != nullptr) {
        // arg-max of the previous step's logits from the per-CTA partials, all clips in flight together
        float bv[4]; int bi[4];
#pragma unroll
        for (int b = 0; b < 4; ++b) { bv[b] = -INFINITY; bi[b] = 0x7fffffff; }
        for (int c = lane; c < a.amax_n; c += 32) {
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            if (b < NB) {
              float v; int ix;
              asm volatile("ld.global.cg.v2.b32 {%0,%1}, [%2];" : "=f"(v), "=r"(ix) : "l"(a.amax_in + (size_t)c * NB + b) : "memory");
              if (v > bv[b] || (v == bv[b] && ix < bi[b])) { bv[b] = v; bi[b] = ix; }
            }
          }
        }
#pragma unroll
        for (int b = 0; b < 4; ++b) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv[b], o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi[b], o);
            if (ov > bv[b] || (ov == bv[b] && oi < bi[b])) { bv[b] = ov; bi[b] = oi; }
          }
          tok[b] = bi[b];
          if (b < NB && blockIdx.x == 0 && tid == 0 && a.tok_out != nullptr) a.tok_out[(long long)b * a.tok_out_stride] = tok[b];
        }
      } else {
#pragma unroll
        for (int b = 0; b < 4; ++b)
          if (b < NB) asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(tok[b]) : "l"(a.tok_in + (long long)b * a.tok_stride) : "memory");
      }
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int t = tok[b] < 0 ? 0 : (tok[b] >= a.vocab ? a.vocab - 1 : tok[b]);
        xg[b] = a.embed + (long long)t * K;
      }
    }
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      if (b < NB) {
#pragma unroll
        for (int u = 0; u < XU; ++u) {
          const int c = tid + u * TC_CONSUMERS;
          if (c < nch)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(xs + (size_t)b * K + c * 8)), "l"(xg[b] + c * 8) : "memory");
        }
      }
    }
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
    // from here on every thread touches only the chunks it copied itself, until the barrier
    if (a.embed != nullptr && a.h_out != nullptr && blockIdx.x == 0) {
      for (int b = 0; b < NB; ++b) {
#pragma unroll
        for (int u = 0; u < XU; ++u) {
          const int c = tid + u * TC_CONSUMERS;
          if (c < nch) *reinterpret_cast<uint4*>(a.h_out + (long long)b * K + c * 8) = *reinterpret_cast<const uint4*>(xs + (size_t)b * K + c * 8);
        }
      }
    }
    if (a.norm_w != nullptr) {
      float ssb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        if (b < NB) {
          // the same per-thread, per-warp and cross-warp summation order as the single-clip path
#pragma unroll
          for (int u = 0; u < XU; ++u) {
            const int c = tid + u * TC_CONSUMERS;
            const uint4 v = (c < nch) ? *reinterpret_cast<const uint4*>(xs + (size_t)b * K + c * 8) : make_uint4(0, 0, 0, 0);
            const float f0 = bf16lo(v.x), f1 = bf16hi(v.x), f2 = bf16lo(v.y), f3 = bf16hi(v.y);
            const float f4 = bf16lo(v.z), f5 = bf16hi(v.z), f6 = bf16lo(v.w), f7 = bf16hi(v.w);
            ssb[b] += f0 * f0 + f1 * f1 + f2 * f2 + f3 * f3 + f4 * f4 + f5 * f5 + f6 * f6 + f7 * f7;
          }
          ssb[b] = warp_sum(ssb[b]);
          if (lane == 0) red[b * TC_CWARPS + warp] = ssb[b];
        }
      }
      cbar();
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        if (b < NB) {
          float tot = 0.f;
#pragma unroll
          for (int w = 0; w < TC_CWARPS; ++w) tot += red[b * TC_CWARPS + w];
          const float rstd = rsqrtf(tot / (float)K + a.eps);
#pragma unroll
          for (int u = 0; u < XU; ++u) {
            const int c = tid + u * TC_CONSUMERS;
            if (c < nch) {
              uint4* px = reinterpret_cast<uint4*>(xs + (size_t)b * K + c * 8);
              const uint4 v = *px;
              const uint4 gwu = *reinterpret_cast<const uint4*>(nw + c * 8);
              uint4 o;
              o.x = bf16x2_mul(gwu.x, pack_bf16x2(bf16lo(v.x) * rstd, bf16hi(v.x) * rstd));
              o.y = bf16x2_mul(gwu.y, pack_bf16x2(bf16lo(v.y) * rstd, bf16hi(v.y) * rstd));
              o.z = bf16x2_mul(gwu.z, pack_bf16x2(bf16lo(v.z) * rstd, bf16hi(v.z) * rstd));
              o.w = bf16x2_mul(gwu.w, pack_bf16x2(bf16lo(v.w) * rstd, bf16hi(v.w) * rstd));
              *px = o;
            }
          }
        }
      }
    }
    cbar();
  } else {
    if (a.norm_w != nullptr) {
      for (int b = 0; b < NB; ++b) {
#pragma unroll
        for (int u = 0; u < XU; ++u) {
          const int c = tid + u * TC_CONSUMERS;
          if (c < nch) *reinterpret_cast<uint4*>(xs + (size_t)b * K + c * 8) = __ldg(reinterpret_cast<const uint4*>(a.norm_w + c * 8));
        }
      }
    }
    float ss = 0.f;
    pdl_wait();                                    // the first activation vector comes from the previous kernel
    if (tid == 0) trace(1);
    for (int b = 0; b < NB; ++b) {                  // one clip after the other (one L2 round trip each)
      bf16* xb = xs + (size_t)b * K;
      const bf16* xg = a.x + (long long)b * a.ldx;
      if (a.embed != nullptr) {
        // fused token-embedding gather: x = embed[token]. The token is either given (first step
        // of a decode loop) or the arg-max of the previous step's logits, whose per-CTA partials
        // every warp reduces for itself (same result in every warp: no barrier needed)
        int tok;
        if (a.amax_in != nullptr) {
          float bv = -INFINITY; int bi = 0x7fffffff;
          for (int c = lane; c < a.amax_n; c += 32) {
            float v; int ix;
            asm volatile("ld.global.cg.v2.b32 {%0,%1}, [%2];" : "=f"(v), "=r"(ix) : "l"(a.amax_in + (size_t)c * NB + b) : "memory");
            if (v > bv || (v == bv && ix < bi)) { bv = v; bi = ix; }
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
          }
          tok = bi;
          if (blockIdx.x == 0 && tid == 0 && a.tok_out != nullptr) a.tok_out[(long long)b * a.tok_out_stride] = tok;
        } else {
          asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(tok) : "l"(a.tok_in + (long long)b * a.tok_stride) : "memory");
        }
        tok = tok < 0 ? 0 : (tok >= a.vocab ? a.vocab - 1 : tok);
        xg = a.embed + (long long)tok * K;
      }
      uint4 xv[XU];
#pragma unroll
      for (int u = 0; u < XU; ++u) {
        const int c = tid + u * TC_CONSUMERS;
        xv[u] = (c < nch) ? ld_cg_v4(xg + c * 8) : make_uint4(0, 0, 0, 0);
      }
      if (a.embed != nullptr && a.h_out != nullptr && blockIdx.x == 0) {
        // the raw embedding row is the residual stream of layer 0 (read by o_proj's epilogue)
#pragma unroll
        for (int u = 0; u < XU; ++u) {
          const int c = tid + u * TC_CONSUMERS;
          if (c < nch) *reinterpret_cast<uint4*>(a.h_out + (long long)b * K + c * 8) = xv[u];
        }
      }
      if (a.norm_w != nullptr) {
        ss = 0.f;
#pragma unroll
        for (int u = 0; u < XU; ++u) {
          const uint4 v = xv[u];
          const float f0 = bf16lo(v.x), f1 = bf16hi(v.x), f2 = bf16lo(v.y), f3 = bf16hi(v.y);
          const float f4 = bf16lo(v.z), f5 = bf16hi(v.z), f6 = bf16lo(v.w), f7 = bf16hi(v.w);
          ss += f0 * f0 + f1 * f1 + f2 * f2 + f3 * f3 + f4 * f4 + f5 * f5 + f6 * f6 + f7 * f7;
        }
        ss = warp_sum(ss);
        if (b > 0) cbar();                          // red[] of the previous clip has been read
        if (lane == 0) red[warp] = ss;
        cbar();
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < TC_CWARPS; ++w) tot += red[w];
        const float rstd = rsqrtf(tot / (float)K + a.eps);
#pragma unroll
        for (int u = 0; u < XU; ++u) {
          const int c = tid + u * TC_CONSUMERS;
          if (c < nch) {
            const uint4 v = xv[u];
            const uint4 gw = *reinterpret_cast<const uint4*>(xb + c * 8);
            uint4 o;
            // w * bf16(x * rstd), the product rounded to bf16 again (LlamaRMSNorm)
            o.x = bf16x2_mul(gw.x, pack_bf16x2(bf16lo(v.x) * rstd, bf16hi(v.x) * rstd));
            o.y = bf16x2_mul(gw.y, pack_bf16x2(bf16lo(v.y) * rstd, bf16hi(v.y) * rstd));
            o.z = bf16x2_mul(gw.z, pack_bf16x2(bf16lo(v.z) * rstd, bf16hi(v.z) * rstd));
            o.w = bf16x2_mul(gw.w, pack_bf16x2(bf16lo(v.w) * rstd, bf16hi(v.w) * rstd));
            *reinterpret_cast<uint4*>(xb + c * 8) = o;
          }
        }
      } else {
#pragma unroll
        for (int u = 0; u < XU; ++u) {
          const int c = tid + u * TC_CONSUMERS;
          if (c < nch) *reinterpret_cast<uint4*>(xb + c * 8) = xv[u];
        }
      }
    }
    cbar();
  }
  if (tid == 0) trace(2);

  for (int grp = 0; grp < ng; ++grp) {
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    for (int kc = 0; kc < nkc; ++kc) {
      const int kb_n = min(TC_KC, K - kc * TC_KC) >> 5;        // 32-wide K blocks in this slot
      mbar_wait(full_bar(slot), par);
      const uint8_t* base = smem + slot * TC_SLOT_BYTES;
#pragma unroll
      for (int t = 0; t < TC_KC / 32 / TC_CWARPS; ++t) {
        const int kb = warp + TC_CWARPS * t;
        if (kb < kb_n) {
          const uint4 wa = *reinterpret_cast<const uint4*>(base + kb * 1024 + lane * 16);        // row g
          const uint4 wb = *reinterpret_cast<const uint4*>(base + kb * 1024 + 512 + lane * 16);  // row g+8
          uint4 xq = make_uint4(0, 0, 0, 0);
          if (g < NB) xq = *reinterpret_cast<const uint4*>(xs + (size_t)g * K + kc * TC_KC + kb * 32 + q * 8);   // column g = clip g
          tc_mma(c, wa.x, wb.x, wa.y, wb.y, xq.x, xq.y);
          tc_mma(c, wa.z, wb.z, wa.w, wb.w, xq.z, xq.w);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(slot));
      advance();
    }
    // the 8 per-warp partials of this row group meet in shared memory (double-buffered: the barrier
    // of the next group orders the reads below before the buffer is written again)
    float* pb = pbuf + (grp & 1) * TC_CWARPS * 16 * 4;
    if (q < 2) {                                    // columns (clips) 2q, 2q+1: rows g (c[0], c[1]) and g+8 (c[2], c[3])
      *reinterpret_cast<float2*>(pb + (warp * 16 + g) * 4 + 2 * q) = make_float2(c[0], c[1]);
      *reinterpret_cast<float2*>(pb + (warp * 16 + g + 8) * 4 + 2 * q) = make_float2(c[2], c[3]);
    }
    cbar();
    if (tid < 64) {                                 // (row, clip) = (tid / 4, tid % 4)
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < TC_CWARPS; ++w) v += pb[w * 64 + tid];
      result[grp * 64 + tid] = v;
    }
  }
  cbar();
  if (tid == 0) trace(3);

  // ---------------- fused epilogue ----------------
  const bool pairs = (mode == TC_MODE_SWIGLU || mode == TC_MODE_QKV);
  const int R = ng * 16;
  const int n_items = (pairs ? R / 2 : R) * NB;     // item = (row or row pair, clip), clip fastest for NB > 1
  for (int it0 = 0; it0 < n_items; it0 += TC_CONSUMERS) {       // uniform trip count: the warps stay converged
    const int it = it0 + tid;
    const int b = (NB == 1) ? 0 : it % NB;
    const int iu = (NB == 1) ? it : it / NB;
    const int rr = pairs ? 2 * iu : iu;
    const int vrow = row0 + rr;
    const bool valid = it < n_items && vrow < N;
    float y = 0.f;                                 // RES / SWIGLU: the output value of this item
    if (valid) {
      const float v0 = result[rr * 4 + b];
      const float v1 = pairs ? result[(rr + 1) * 4 + b] : 0.f;
      if (mode == TC_MODE_RES) {
        y = bf16r(v0);
        if (p.res != nullptr) {                    // written by an earlier kernel: read through L2
          unsigned short rv;
          asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(rv) : "l"(p.res + (long long)b * p.ldr + vrow) : "memory");
          y += __uint_as_float((uint32_t)rv << 16);
        }
        p.out[(long long)b * p.ldo + vrow] = __float2bfloat16_rn(y);
      } else if (mode == TC_MODE_LOGITS) {
        if (p.logits != nullptr) p.logits[(long long)b * p.ldl + vrow] = bf16r(v0);
      } else if (mode == TC_MODE_SWIGLU) {
        const float gt = bf16r(v0);
        const float sg = bf16r(__fdividef(gt, 1.0f + __expf(-gt)));
        y = sg * bf16r(v1);
        p.out[(long long)b * p.ldo + (vrow >> 1)] = __float2bfloat16_rn(y);
      } else {  // TC_MODE_QKV: vrow = (which*H + head)*128 + 2*d
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
  if (mode == TC_MODE_LOGITS && a.amax_out != nullptr) {
    // per-CTA partial arg-max over this CTA's rows (bf16-rounded logits, lowest index wins ties);
    // the consumer of the partials keeps the lowest index across CTAs as well
    for (int b = 0; b < NB; ++b) {
      float bv = -INFINITY; int bi = 0x7fffffff;
      for (int rr = tid; rr < R; rr += TC_CONSUMERS) {
        const int vrow = row0 + rr;
        if (vrow < N) {
          const float v = bf16r(result[rr * 4 + b]);
          if (v > bv) { bv = v; bi = vrow; }          // rr ascending: the first maximum is kept
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      cbar();                                          // pbuf is free (and the previous clip's slots read)
      if (lane == 0) { pbuf[2 * warp] = bv; pbuf[2 * warp + 1] = __int_as_float(bi); }
      cbar();
      if (tid == 0) {
#pragma unroll
        for (int w = 1; w < TC_CWARPS; ++w) {
          const float ov = pbuf[2 * w]; const int oi = __float_as_int(pbuf[2 * w + 1]);
          if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        ArgmaxPart ap; ap.v = bv; ap.idx = bi;
        a.amax_out[(size_t)blockIdx.x * NB + b] = ap;
      }
    }
  }
  if (tid == 0) {
    trace(4);
    if (p.trace != nullptr) p.trace[(size_t)blockIdx.x * 8 + 7] = ((unsigned long long)mode << 32) | (unsigned)N;
  }
}

// row-major W[N][K] -> tiled copy. One thread per 16-byte chunk of the output.
__global__ void gemv_tc_repack_kernel(const bf16* __restrict__ W, bf16* __restrict__ dst, int N, int K, int qkv) {
  const size_t chunks_per_group = (size_t)2 * K;                      // 16 rows x K x 2 B / 16 B
  const size_t n_chunks = (size_t)((N + 15) >> 4) * chunks_per_group;
  for (size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x; o < n_chunks; o += (size_t)gridDim.x * blockDim.x) {
    const int grp = (int)(o / chunks_per_group);
    const size_t off = (o - (size_t)grp * chunks_per_group) * 16;     // byte offset inside the group
    const int kc = (int)(off / ((size_t)TC_KC * 32));
    const int within = (int)(off - (size_t)kc * TC_KC * 32);
    const int kb = within >> 10, r = within & 1023;
    const int half = r >> 9, l = (r & 511) >> 4;
    const int row = grp * 16 + (l >> 2) + 8 * half;
    const int k = kc * TC_KC + kb * 32 + (l & 3) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row < N) {
      const long long src_row = qkv ? qkv_row(row) : (long long)row;
      v = *reinterpret_cast<const uint4*>(W + src_row * K + k);
    }
    *reinterpret_cast<uint4*>(dst + o * 8) = v;
  }
}

// shared-memory plan on `grid` CTAs; returns the slot count (0 = does not fit)
int plan(int nb, int N, int K, bool norm, int ring_slots, int grid, size_t* smem_bytes, int* x_elems, int* r_cap) {
  if (K % 32 != 0 || K > 14336) return 0;
  const int xe = K * (nb + ((nb > 1 && norm) ? 1 : 0));   // x buffer: nb vectors (+ the parked norm weights when nb > 1)
  const int rmax = (((N + 15) / 16 + grid - 1) / grid) * 16;
  int want = ring_slots > TC_DEFAULT_SLOTS ? ring_slots : TC_DEFAULT_SLOTS;
  const size_t fixed = (size_t)xe * 2 + (size_t)(2 * TC_CWARPS * 16 + rmax) * 4 * 4 + 4 * TC_CWARPS * 4 + 2 * TC_MAX_SLOTS * 8 + 128;
  static const int env_slots = getenv("VCL_GEMV_TC_SLOTS") ? atoi(getenv("VCL_GEMV_TC_SLOTS")) : 0;
  static const size_t budget = getenv("VCL_GEMV_TC_SMEM_KB") ? (size_t)atoi(getenv("VCL_GEMV_TC_SMEM_KB")) * 1024 : (size_t)TC_SMEM_BUDGET;
  if (fixed + 4 * (size_t)TC_SLOT_BYTES > (nb > 1 ? (size_t)212 * 1024 : budget)) return 0;
  // a launch may ask for a deeper ring (the projection after the attention kernel sits resident with
  // nothing to do but prefetch); the hard limit leaves room for the attention CTAs
  const size_t limit = (want > TC_DEFAULT_SLOTS || nb > 1) ? (size_t)212 * 1024 : budget;   // several clips: x takes the room
  int slots = (int)((limit - fixed) / TC_SLOT_BYTES);
  if (want > TC_MAX_SLOTS) want = TC_MAX_SLOTS;
  if (slots > want) slots = want;
  if (env_slots > 0 && env_slots < slots) slots = env_slots;
  *smem_bytes = (size_t)slots * TC_SLOT_BYTES + fixed;
  *x_elems = xe; *r_cap = rmax;
  return slots;
}

// VCL_TC_TRACE: every launch writes 8 timestamps per CTA into the next record of a device buffer;
// vcl_debug_tc_trace_dump() (below) writes the records to a file. Debug aid for eager runs.
constexpr int TC_TRACE_RECORDS = 512;
unsigned long long* g_trace = nullptr;
int g_trace_next = 0;

int tc_launch(TcParams p, cudaStream_t stream) {
  const GemvArgs& a = p.a;
  VCL_REQUIRE(gemv_tc_fits(a.B, a.N, a.K, a.norm_w != nullptr),
              "gemv_tc: B=%d N=%d K=%d is outside the kernel's range (1..4 clips, K a multiple of 32 and <= 14336)",
              a.B, a.N, a.K);
  VCL_REQUIRE(a.W_tiled != nullptr && (uintptr_t)a.W_tiled % 16 == 0 && a.ldx % 8 == 0 &&
              (a.embed != nullptr || (uintptr_t)a.x % 16 == 0), "gemv_tc: operands must be 16-byte aligned");
  const int grid = gemv_tc_grid(a.N);
  size_t smem = 0;
  p.n_slots = plan(a.B, a.N, a.K, a.norm_w != nullptr, a.ring_slots, grid, &smem, &p.x_elems, &p.r_cap);
  static const bool tracing = getenv("VCL_TC_TRACE") != nullptr;
  if (tracing) {
    const size_t rec = (size_t)device_num_sms() * 8;
    if (g_trace == nullptr) {
      VCL_CUDA_OK(cudaMalloc(&g_trace, TC_TRACE_RECORDS * rec * sizeof(unsigned long long)));
      VCL_CUDA_OK(cudaMemset(g_trace, 0, TC_TRACE_RECORDS * rec * sizeof(unsigned long long)));
    }
    p.trace = g_trace + (size_t)(g_trace_next % TC_TRACE_RECORDS) * rec;
    ++g_trace_next;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, gemv_tc_kernel, p));
  count_launches(1);
  return 0;
}

TcParams tc_params(const GemvArgs& g, int mode) {
  TcParams p = {};
  p.a = g; p.mode = mode;
  return p;
}

}  // namespace

extern "C" int vcl_debug_tc_trace_dump(const char* path) {
  if (g_trace == nullptr) return -1;
  const size_t n = (size_t)TC_TRACE_RECORDS * device_num_sms() * 8;
  std::vector<unsigned long long> host(n + 2);
  VCL_CUDA_OK(cudaDeviceSynchronize());
  VCL_CUDA_OK(cudaMemcpy(host.data() + 2, g_trace, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  host[0] = (unsigned long long)g_trace_next; host[1] = (unsigned long long)device_num_sms();
  FILE* f = fopen(path, "wb");
  if (f == nullptr) return -2;
  fwrite(host.data(), sizeof(unsigned long long), n + 2, f);
  fclose(f);
  return 0;
}

int init_gemv_tc_kernels() {
  VCL_CUDA_OK(cudaFuncSetAttribute(gemv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
  return 0;
}

// one CTA per SM, but none without a row group
int gemv_tc_grid(int N) {
  const int n_groups = (N + 15) / 16, sms = device_num_sms();
  return n_groups < sms ? n_groups : sms;
}

bool gemv_tc_fits(int B, int N, int K, bool norm) {
  if (B < 1 || B > 4 || N < 1) return false;
  size_t smem = 0; int xe = 0, rc = 0;
  return plan(B, N, K, norm, 0, gemv_tc_grid(N), &smem, &xe, &rc) >= 4;
}

size_t gemv_tc_tiled_elems(int N, int K) { return (size_t)((N + 15) / 16) * 16 * K; }

int launch_gemv_tc_repack(const bf16* W, bf16* dst, int N, int K, bool qkv_pairs, cudaStream_t stream) {
  VCL_REQUIRE(K % 32 == 0, "gemv_tc repack: K=%d must be a multiple of 32", K);
  VCL_REQUIRE(!qkv_pairs || N % 128 == 0, "gemv_tc repack: q/k/v rows must come in heads of 128 (N=%d)", N);
  gemv_tc_repack_kernel<<<device_num_sms() * 8, 256, 0, stream>>>(W, dst, N, K, qkv_pairs ? 1 : 0);
  VCL_CUDA_OK(cudaGetLastError());
  return 0;
}

int launch_gemv_tc_residual(const GemvArgs& g, bf16* out, long long ldo, const bf16* res, long long ldr,
                            cudaStream_t stream) {
  TcParams p = tc_params(g, TC_MODE_RES);
  p.out = out; p.ldo = ldo; p.res = res; p.ldr = ldr;
  return tc_launch(p, stream);
}

int launch_gemv_tc_swiglu(const GemvArgs& g, bf16* out, long long ldo, cudaStream_t stream) {
  VCL_REQUIRE(g.N % 2 == 0, "gemv swiglu: N must be even (interleaved gate/up rows)");
  TcParams p = tc_params(g, TC_MODE_SWIGLU);
  p.out = out; p.ldo = ldo;
  return tc_launch(p, stream);
}

int launch_gemv_tc_qkv_rope(const GemvArgs& g, bf16* q_out, long long ldq, bf16* kcache, bf16* vcache,
                            const bf16* cos_t, const bf16* sin_t, int H, int s_max, int pos, cudaStream_t stream,
                            const int* pos_dev) {
  VCL_REQUIRE(g.N == 3 * H * 128, "gemv_tc qkv: N=%d != 3*H*128", g.N);
  VCL_REQUIRE(g.embed == nullptr || (g.vocab > 0 && (g.tok_in != nullptr || (g.amax_in != nullptr && g.amax_n > 0))),
              "gemv_tc qkv: the fused embedding gather needs a token source");
  TcParams p = tc_params(g, TC_MODE_QKV);
  p.q_out = q_out; p.ldq = ldq; p.kcache = kcache; p.vcache = vcache;
  p.cos_t = cos_t; p.sin_t = sin_t; p.H = H; p.s_max = s_max; p.pos = pos; p.pos_dev = pos_dev;
  return tc_launch(p, stream);
}

int launch_gemv_tc_logits(const GemvArgs& g, float* logits, long long ldl, cudaStream_t stream) {
  TcParams p = tc_params(g, TC_MODE_LOGITS);
  p.logits = logits; p.ldl = ldl;
  return tc_launch(p, stream);
}

}  // namespace vcl

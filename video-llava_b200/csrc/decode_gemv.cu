// Decode projections for 1..64 clips: out[b][n] = x[b] . W[n, :], one kernel per weight matrix, the weights
// streamed ONCE per launch. Two kernels share the streaming machinery and the epilogues:
//   gemv_tc_kernel            1..4 clips, the activation vectors staged in shared memory
//   gemv_tcw_kernel<NG, CG>   5..64 clips, the activations streamed window by window next to the weights, the
//                             clips split into CG groups of 16 across the consumer warps (CG = 1, 2, 4)
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
// Common structure (one CTA per SM, at most one per 16-row group; 9 warps, a ring of 16 KB slots):
//   warp 8      producer: walks this CTA's 16-row groups and 512-k chunks and fills the ring with one bulk
//               copy per slot. Both kernels read a decode-only copy of the matrix that the weight loader
//               lays out slot by slot (gemv_tc_repack_kernel): [16-row group][K chunk][32-wide K block]
//               [row half][lane] x 16 bytes, i.e. already in mma.sync A-fragment order. Weights never
//               depend on the previous kernel, so the producer starts BEFORE the dependency wait.
//   warps 0-7   consumers: per slot, every warp takes every eighth 32-wide K block, two conflict-free
//               LDS.128 for the A fragments (lane l reads bytes [16 l, 16 l + 16) of each 512-byte row
//               half) and two m16n8k16 MMAs per column block of 8 clips (clip b = column b of the B
//               operand). A slot is free again ~100 cycles after it landed, so almost the whole ring is
//               in flight from HBM at any time. The 8 per-warp partials meet in shared memory and the
//               fused epilogues (RoPE + KV append, SwiGLU, residual, logits) run once at the end.
//
// gemv_tc_kernel (1..4 clips): the consumers stage every clip's activation vector in shared memory (bf16,
// optionally RMS-normalised, or gathered from the token-embedding table) and walk the ring group by group;
// fp32 accumulators live across the K chunks of a row group, the per-warp partials meet after every group.
//
// gemv_tcw_kernel<NG, CG> (5..64 clips):
//   * the activations no longer fit in shared memory next to the ring (16 x 11008 x 2 B = 352 KB for
//     down_proj), so the K dimension is walked chunk-major: for every 512-wide K chunk the producer first
//     copies that WINDOW of the (already normalised) activations and then the slots of that chunk for all
//     row groups of the CTA. The slots are contiguous 16 KB blocks whatever the order they are visited in,
//     so the same weight copy serves both kernels. The activations are kept in global memory window-major
//     ("xwin", kernels.h), so that a window is ONE contiguous bulk copy -- the copy engine retires ~23
//     copies per microsecond and SM whatever their size, sixteen 1 KB row copies per chunk made o_proj /
//     down_proj copy-rate bound -- and its rows arrive already padded to 1088 B, which makes the B-fragment
//     loads of the 8 clips of an MMA bank-conflict free. Whoever produces an input of this kernel writes
//     that layout: the decode-path RMSNorm (launch_xwin_norm), the decode attention kernel and this
//     kernel's own SwiGLU epilogue.
//   * the 8 consumer warps are CG clip groups of 16 (clip group cg = columns 16 cg .. 16 cg + 15 of the MMA B
//     operand) x KP = 8 / CG K phases (warp kp of a group takes the 32-wide K blocks kp, kp + KP, ...): CG = 1
//     for 5..16 clips, 2 for 17..32, 4 for 33..64. An A fragment is loaded by CG warps.
//   * the accumulators of ALL row groups of the CTA (up to NG groups x 2 column blocks x 4 registers per warp)
//     and the B fragments of the warp's K blocks stay in registers across the K chunks; the KP partial tiles of
//     a group meet once, at the end, in the (then idle) shared memory. A 9-warp kernel has at most 168 registers
//     per thread (3 warps share a sub-partition's 16K), so the largest instances without spills hold NG = 14 /
//     10 / 6 row groups at CG = 1 / 2 / 4. A matrix with more row groups per SM is streamed by consecutive
//     launches over near-equal row slices; r0 is the slice's first row (the weights and row scales of `a` start
//     there, the epilogue addresses rows r0 + local row).
//   * a warp per row group (no reduction at all) keeps a slot held for ~1000 cycles by its one consumer, so
//     only a few of the ring slots are in flight; per-row window copies make the copy engine the limit.
//
// Weight formats (GemvArgs): both kernels are templates over the format of the slot-ordered copy.
//   W_BF16  the bf16 copy above.
//   W_FP8   E4M3 codes q in the SAME order, one byte per weight (a 512-k slot is 8 KB; the ring keeps its size
//           and holds twice as many slots), plus a power-of-two scale 2^e per row (w_scale). The consumers turn
//           the codes into exactly the bf16 A fragments of q (e4m3x2_bf16x2), issue the same MMAs in the same k
//           order and warp split, and multiply each row's fp32 dot product, after the cross-warp sum, by 2^e.
//           A power-of-two factor commutes with every fp32 rounding of those sums (no under- or overflow), so the
//           result equals the bf16 kernel's on W~ = q * 2^e bit for bit (DESIGN.md section 3). The load-time
//           quantizer (gemv_quantize_fp8_kernel) writes W~ over the row-major matrix for every other path.
//
// Rounding points (reference: transformers/models/llama/modeling_llama.py:53-67 RMSNorm, :124-168 RoPE,
// :171-184 MLP, :325,331 residuals): the normalised activation w * bf16(x * rstd) is rounded to bf16, every
// projection is rounded to bf16 before its epilogue, and so are the RoPE products, silu(gate) and the
// residual sum; logits are kept bf16-rounded in fp32. The epilogue functions below are the one place
// where these roundings are written down for both kernels.
#include "common.cuh"
#include "kernels.h"

#include <cuda_fp8.h>

#include <stdio.h>
#include <stdlib.h>

#include <vector>

namespace vcl {

namespace {

constexpr int CWARPS = 8;                           // consumer warps
constexpr int CONSUMERS = CWARPS * 32;
constexpr int THREADS = CONSUMERS + 32;             // + the producer warp
constexpr int KC = 512;                             // k elements per slot
constexpr int SLOT_BYTES = 16 * KC * 2;             // 16 KB, one bulk copy
constexpr int SLOTS = 8;                            // ring depth (gemv_tc: at most; not re-tuned on the H100)

// gemv_tc: shared-memory limit of a launch. One clip stays within 160 KB, so that the rest of the SM
// stays free for the attention kernel's CTAs, which launch early (PDL); several clips need the room for
// their activation vectors.
constexpr int TC_SMEM_ONE_CLIP = 160 * 1024;
constexpr int TC_SMEM_CLIPS = 212 * 1024;

// the ring of each weight format: bytes per weight, per slot, and slots in the same 128 KB
constexpr int W_BF16 = 0, W_FP8 = 1;
template <int FMT> struct Ring {
  static constexpr int EB = FMT == W_FP8 ? 1 : 2;
  static constexpr int SLOT = 16 * KC * EB;
  static constexpr int NSLOT = SLOTS * 2 / EB;
};

// gemv_tcw: shared-memory plan of CG clip groups (not swept on the H100): a ring of RING bytes, NWIN activation
// windows of 16 CG clips in flight, then the barriers (full / empty per slot and per window)
//   CG = 1: 128 KB ring (8 bf16 / 16 fp8 slots), 4 windows of 16 clips. With two windows, a CTA that owns 1-2 row
//           groups (o_proj, down_proj) waited an L2 round trip for a window every second chunk.
//   CG = 2:  80 KB ring (5 / 10 slots), 4 windows of 32 clips
//   CG = 4:  80 KB ring (5 / 10 slots), 2 windows of 64 clips
constexpr int TW_XROW = XWIN_PITCH * 2;             // 1088 bytes per activation row of a window
template <int CG, int FMT> struct TwPlan {
  static constexpr int RING = (CG == 1 ? 8 : 5) * SLOT_BYTES;
  static constexpr int NSLOT = RING / Ring<FMT>::SLOT;
  static constexpr int NWIN = CG == 4 ? 2 : 4;      // a power of two
  static constexpr int XBUF = 16 * CG * TW_XROW;
  static constexpr int XAREA = NWIN * XBUF;
  static constexpr int BARS = CG == 1 && FMT == W_BF16 ? 256 : 512;
  static constexpr int SMEM = RING + XAREA + BARS;
  static_assert(2 * (NSLOT + NWIN) * 8 <= BARS, "barriers");
};

struct TcParams {
  GemvArgs a;                       // a.B clips (1..4) are the columns of the MMA B operand
  GemvEpilogue e;
  int n_slots;
  int x_elems;                      // activation buffer (elements)
  int r_cap;                        // rows one CTA owns at most (result buffer)
  unsigned long long* trace;        // optional [grid][8] timestamps (VCL_TC_TRACE)
};

// ---------------------------------------------------------------------------------------------
// shared device code
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                         uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// Two E4M3 codes (bytes 0, 1 of w with SEL 0x9180, bytes 2, 3 with 0xB3A2) -> the bf16 pair of equal value, the
// lower byte in the lower half. prmt lays out [code, sign x 8] per half; shifted by 4 and masked, the half holds
// the code's sign, its 4-bit exponent field in the low bits of bf16's 8-bit one and its 3 mantissa bits on top
// of bf16's 7, i.e. the bf16 number code * 2^-120 (a normal code stays normal, a subnormal one stays subnormal,
// +-0 stays +-0). The multiplication by 2^120 is exact for every finite code (NaN codes never occur).
template <uint32_t SEL>
__device__ __forceinline__ uint32_t e4m3x2_bf16x2(uint32_t w) {
  uint32_t t, r;
  asm("prmt.b32 %0, %1, 0, %2;" : "=r"(t) : "r"(w), "n"(SEL));
  t = (t << 4) & 0x87f087f0u;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(t), "r"(0x7b807b80u));   // 0x7b80 = bf16(2^120)
  return r;
}
// The A fragments of one 32-wide K block of a slot, rows g (wa) and g + 8 (wb): 8 consecutive k per lane and row
// half, k order (0,1) (2,3) (4,5) (6,7) in .x .y .z .w
template <int FMT>
__device__ __forceinline__ void load_a(const uint8_t* base, int kb, int lane, uint4& wa, uint4& wb) {
  if constexpr (FMT == W_FP8) {
    const uint2 ca = *reinterpret_cast<const uint2*>(base + kb * 512 + lane * 8);
    const uint2 cb = *reinterpret_cast<const uint2*>(base + kb * 512 + 256 + lane * 8);
    wa = make_uint4(e4m3x2_bf16x2<0x9180>(ca.x), e4m3x2_bf16x2<0xB3A2>(ca.x), e4m3x2_bf16x2<0x9180>(ca.y),
                    e4m3x2_bf16x2<0xB3A2>(ca.y));
    wb = make_uint4(e4m3x2_bf16x2<0x9180>(cb.x), e4m3x2_bf16x2<0xB3A2>(cb.x), e4m3x2_bf16x2<0x9180>(cb.y),
                    e4m3x2_bf16x2<0xB3A2>(cb.y));
  } else {
    wa = *reinterpret_cast<const uint4*>(base + kb * 1024 + lane * 16);          // row g
    wb = *reinterpret_cast<const uint4*>(base + kb * 1024 + 512 + lane * 16);    // row g + 8
  }
}
// the weight bytes of a launch and the fp32 row scale (1 for bf16 weights)
template <int FMT> __device__ __forceinline__ const uint8_t* weight_bytes(const GemvArgs& a) {
  if constexpr (FMT == W_FP8) return a.W_fp8;
  else return reinterpret_cast<const uint8_t*>(a.W_tiled);
}
template <int FMT> __device__ __forceinline__ float row_scaled(const GemvArgs& a, int row, float v) {
  if constexpr (FMT == W_FP8) return v * __ldg(a.w_scale + row);
  else return v;
}
__device__ __forceinline__ void cbar() {            // barrier among the consumer warps only
  asm volatile("bar.sync 1, %0;" ::"r"(CONSUMERS) : "memory");
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
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

// This CTA's row groups: contiguous blocks of 16-row groups per CTA, sizes differing by at most one group,
// the larger shares spread evenly over the grid. Returns the count, grp_begin the first group.
__device__ __forceinline__ int cta_row_groups(int N, int& grp_begin) {
  const int n_groups = (N + 15) >> 4;
  grp_begin = (int)(((long long)blockIdx.x * n_groups) / gridDim.x);
  return (int)(((long long)(blockIdx.x + 1) * n_groups) / gridDim.x) - grp_begin;
}

// arg-max with the lowest index winning ties: (v, i) takes (ov, oi) if that is larger or equal at a lower index
__device__ __forceinline__ void argmax_take(float& v, int& i, float ov, int oi) {
  if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
}
__device__ __forceinline__ void warp_argmax(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) argmax_take(v, i, __shfl_xor_sync(0xffffffffu, v, o), __shfl_xor_sync(0xffffffffu, i, o));
}

// ---- epilogue items: the fp32 dot product(s) of one row (pair) and clip b -> outputs ----
// RES: out[b][row] = bf16(bf16(v) + res[b][row])
__device__ __forceinline__ void epi_residual(const GemvEpilogue& e, int b, int row, float v) {
  float y = bf16r(v);
  if (e.res != nullptr) {                    // written by an earlier kernel: read through L2
    unsigned short rv;
    asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(rv) : "l"(e.res + (long long)b * e.ldr + row) : "memory");
    y += __uint_as_float((uint32_t)rv << 16);
  }
  e.out[(long long)b * e.ldo + row] = __float2bfloat16_rn(y);
}
// LOGITS: logits[b][row] = bf16-rounded v (null: not stored)
__device__ __forceinline__ void epi_logit(const GemvEpilogue& e, int b, int row, float v) {
  if (e.logits != nullptr) e.logits[(long long)b * e.ldl + row] = bf16r(v);
}
// SWIGLU: rows (row, row + 1) = (gate_j, up_j) -> out[b][j] = silu(gate) * up, row-major or in the xwin
// layout of nb clips
__device__ __forceinline__ void epi_swiglu(const GemvEpilogue& e, int b, int row, int nb, float gate, float up) {
  const float gt = bf16r(gate);
  const float sg = bf16r(act_sigmoid_div(gt, gt));
  const int col = row >> 1;
  const long long o = e.out_xwin ? (long long)xwin_offset(b, col, nb) : (long long)b * e.ldo + col;
  e.out[o] = __float2bfloat16_rn(sg * bf16r(up));
}
// QKV: row = (which*H + head)*128 + 2*d holds dims (d, d + 64) of q, k or v (RoPE pairs adjacent); q and k are
// rotated by the angle of max(col - floor, 0), q goes to q_out, k and v to the cache at column col. The caller
// passes clip b's column (decode_col) and key floor n_pad[b], so that both loads are issued before the epilogue's
// dependent chain (kernels.h: decode positions).
__device__ __forceinline__ int decode_col(const GemvEpilogue& e, int b) {
  return e.pos + (e.pos_dev != nullptr ? __ldg(e.pos_dev + b) : 0);
}
__device__ __forceinline__ void epi_qkv_rope(const GemvEpilogue& e, int b, int row, int col, int floor, float v0,
                                             float v1) {
  const int hr = row >> 7;
  const int which = hr / e.H, head = hr - which * e.H;
  const int d = (row & 127) >> 1;
  const float lo = bf16r(v0), hi = bf16r(v1);
  // a paged cache: clip b is cache slot b, its column col in block table[b][col / 128]
  const long long coff = e.pages.table != nullptr ? kv_paged_off(e.pages, b, head, col)
                                                  : (((long long)b * e.H + head) * e.s_max + col) * 128;
  if (which == 2) {
    e.vcache[coff + d] = __float2bfloat16_rn(lo);
    e.vcache[coff + d + 64] = __float2bfloat16_rn(hi);
  } else {
    const int rpos = max(col - floor, 0);
    const float cs = __bfloat162float(e.cos_t[(long long)rpos * 64 + d]);
    const float sn = __bfloat162float(e.sin_t[(long long)rpos * 64 + d]);
    const float olo = bf16r(lo * cs) + bf16r(-hi * sn);
    const float ohi = bf16r(hi * cs) + bf16r(lo * sn);
    if (which == 0) {
      e.q_out[(long long)b * e.ldq + head * 128 + d] = __float2bfloat16_rn(olo);
      e.q_out[(long long)b * e.ldq + head * 128 + d + 64] = __float2bfloat16_rn(ohi);
    } else {
      e.kcache[coff + d] = __float2bfloat16_rn(olo);
      e.kcache[coff + d + 64] = __float2bfloat16_rn(ohi);
    }
  }
}

// virtual q/k/v row -> weight row: the rows of a RoPE pair (d, d+64) are made adjacent (2p, 2p+1)
__device__ __forceinline__ long long qkv_row(int v) {
  return (long long)(v >> 7) * 128 + ((v & 127) >> 1) + (((v & 127) & 1) << 6);
}

// ---------------------------------------------------------------------------------------------
// 1..4 clips
// ---------------------------------------------------------------------------------------------
template <int FMT>
__global__ void __launch_bounds__(THREADS, 2) gemv_tc_kernel(const TcParams p) {
  using RG = Ring<FMT>;
  extern __shared__ __align__(128) uint8_t smem[];
  // layout: ring[n_slots] | x[nb][K] bf16 (+ norm weights [K]) | pbuf[2][CWARPS][16][4] | result[r_cap][4] fp32
  //         | red | barriers
  const int n_slots = p.n_slots;
  bf16* xs = reinterpret_cast<bf16*>(smem + (size_t)n_slots * RG::SLOT);
  float* pbuf = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(xs) + (size_t)p.x_elems * 2);
  float* result = pbuf + 2 * CWARPS * 16 * 4;
  float* red = result + p.r_cap * 4;
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + 4 * CWARPS);
  const uint32_t ring0 = smem_u32(smem);
  const uint32_t bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (RG::NSLOT + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  auto trace = [&](int ev) {
    if (p.trace != nullptr) p.trace[(size_t)blockIdx.x * 8 + ev] = globaltimer_ns();
  };
  if (tid == 0) {
    trace(0);
    for (int s = 0; s < n_slots; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), CWARPS); }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_launch_dependents();                           // the next kernel (attention) may become resident

  const GemvArgs& a = p.a;
  const GemvEpilogue& e = p.e;
  int slot = 0;
  uint32_t par = 0;
  auto advance = [&]() { if (++slot == n_slots) { slot = 0; par ^= 1u; } };

  if (warp == CWARPS) {
    // =============================== producer ===============================
    // never waits for the consumers' epilogue or activation fetch: HBM keeps streaming meanwhile
    if (lane == 0) {
      const int K = a.K, nkc = (K + KC - 1) / KC;
      int grp_begin;
      const int ng = cta_row_groups(a.N, grp_begin);
      trace(5);
      for (int g = 0; g < ng; ++g) {
        const uint8_t* src = weight_bytes<FMT>(a) + (size_t)(grp_begin + g) * 16 * K * RG::EB;
        for (int kc = 0; kc < nkc; ++kc) {
          const uint32_t bytes = (uint32_t)min(KC, K - kc * KC) * (16u * RG::EB);    // 16 rows
          mbar_wait(empty_bar(slot), par ^ 1u);
          mbar_arrive_expect_tx(full_bar(slot), bytes);
          bulk_g2s(ring0 + slot * RG::SLOT, src + (size_t)kc * KC * 16 * RG::EB, bytes, full_bar(slot));
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
  const int K = a.K, N = a.N, mode = e.mode;
  const int nkc = (K + KC - 1) / KC;
  const int nch = K >> 3;
  int grp_begin;
  const int ng = cta_row_groups(N, grp_begin);
  const int row0 = grp_begin * 16;
  // Activation vectors -> shared memory (bf16), RMS-normalised when the layer norm is fused. The norm
  // weights (constants) are parked in shared memory first; the dependent latency is one L2 round trip.
  const int NB = a.B;
  if (NB > 1) {
    // ---- 2-4 clips: every clip's vector is fetched at once (cp.async.cg straight into the x buffer: ONE L2
    // round trip for the launch instead of one per clip), then normalised in place. The norm weights (the
    // same for every clip) are parked behind the x buffer.
    bf16* nw = xs + (size_t)NB * K;                   // the plan reserves K more elements for launches with a norm
    if (a.norm_w != nullptr) {
#pragma unroll
      for (int u = 0; u < XU; ++u) {
        const int c = tid + u * CONSUMERS;
        if (c < nch) *reinterpret_cast<uint4*>(nw + c * 8) = __ldg(reinterpret_cast<const uint4*>(a.norm_w + c * 8));
      }
    }
    pdl_wait();                                       // the activation vectors come from the previous kernel
    if (tid == 0) trace(1);
    const bf16* xg[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) xg[b] = a.x + (long long)(b < NB ? b : 0) * a.ldx;
    if (a.embed != nullptr) {
      // fused token-embedding gather: x = embed[token]. The token is either given (first step of a decode
      // loop) or the arg-max of the previous step's logits, whose per-CTA partials every warp reduces for
      // itself (same result in every warp: no barrier needed), all clips in flight together
      int tok[4] = {0, 0, 0, 0};
      if (a.amax_in != nullptr) {
        float bv[4]; int bi[4];
#pragma unroll
        for (int b = 0; b < 4; ++b) { bv[b] = -INFINITY; bi[b] = 0x7fffffff; }
        for (int c = lane; c < a.amax_n; c += 32) {
#pragma unroll
          for (int b = 0; b < 4; ++b) {
            if (b < NB) {
              float v; int ix;
              asm volatile("ld.global.cg.v2.b32 {%0,%1}, [%2];" : "=f"(v), "=r"(ix) : "l"(a.amax_in + (size_t)c * NB + b) : "memory");
              argmax_take(bv[b], bi[b], v, ix);
            }
          }
        }
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          warp_argmax(bv[b], bi[b]);
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
          const int c = tid + u * CONSUMERS;
          if (c < nch)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(xs + (size_t)b * K + c * 8)), "l"(xg[b] + c * 8) : "memory");
        }
      }
    }
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
    // from here on every thread touches only the chunks it copied itself, until the barrier
    if (a.embed != nullptr && a.h_out != nullptr && blockIdx.x == 0) {
      // the raw embedding row is the residual stream of layer 0 (read by o_proj's epilogue)
      for (int b = 0; b < NB; ++b) {
#pragma unroll
        for (int u = 0; u < XU; ++u) {
          const int c = tid + u * CONSUMERS;
          if (c < nch) *reinterpret_cast<uint4*>(a.h_out + (long long)b * K + c * 8) = *reinterpret_cast<const uint4*>(xs + (size_t)b * K + c * 8);
        }
      }
    }
    if (a.norm_w != nullptr) {
      float ssb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        if (b < NB) {
#pragma unroll
          for (int u = 0; u < XU; ++u) {
            const int c = tid + u * CONSUMERS;
            const uint4 v = (c < nch) ? *reinterpret_cast<const uint4*>(xs + (size_t)b * K + c * 8) : make_uint4(0, 0, 0, 0);
            const float f0 = bf16lo(v.x), f1 = bf16hi(v.x), f2 = bf16lo(v.y), f3 = bf16hi(v.y);
            const float f4 = bf16lo(v.z), f5 = bf16hi(v.z), f6 = bf16lo(v.w), f7 = bf16hi(v.w);
            ssb[b] += f0 * f0 + f1 * f1 + f2 * f2 + f3 * f3 + f4 * f4 + f5 * f5 + f6 * f6 + f7 * f7;
          }
          ssb[b] = warp_sum(ssb[b]);
          if (lane == 0) red[b * CWARPS + warp] = ssb[b];
        }
      }
      cbar();
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        if (b < NB) {
          float tot = 0.f;
#pragma unroll
          for (int w = 0; w < CWARPS; ++w) tot += red[b * CWARPS + w];
          const float rstd = rsqrtf(tot / (float)K + a.eps);
#pragma unroll
          for (int u = 0; u < XU; ++u) {
            const int c = tid + u * CONSUMERS;
            if (c < nch) {
              uint4* px = reinterpret_cast<uint4*>(xs + (size_t)b * K + c * 8);
              const uint4 v = *px;
              const uint4 gwu = *reinterpret_cast<const uint4*>(nw + c * 8);
              uint4 o;
              // w * bf16(x * rstd), the product rounded to bf16 again (LlamaRMSNorm)
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
  } else {
    // ---- 1 clip: the vector is loaded into registers and normalised on its way to shared memory, where the
    // norm weights were parked. The same per-thread, per-warp and cross-warp summation order as above.
    if (a.norm_w != nullptr) {
#pragma unroll
      for (int u = 0; u < XU; ++u) {
        const int c = tid + u * CONSUMERS;
        if (c < nch) *reinterpret_cast<uint4*>(xs + c * 8) = __ldg(reinterpret_cast<const uint4*>(a.norm_w + c * 8));
      }
    }
    pdl_wait();
    if (tid == 0) trace(1);
    const bf16* xg = a.x;
    if (a.embed != nullptr) {
      int tok;
      if (a.amax_in != nullptr) {
        float bv = -INFINITY; int bi = 0x7fffffff;
        for (int c = lane; c < a.amax_n; c += 32) {
          float v; int ix;
          asm volatile("ld.global.cg.v2.b32 {%0,%1}, [%2];" : "=f"(v), "=r"(ix) : "l"(a.amax_in + c) : "memory");
          argmax_take(bv, bi, v, ix);
        }
        warp_argmax(bv, bi);
        tok = bi;
        if (blockIdx.x == 0 && tid == 0 && a.tok_out != nullptr) a.tok_out[0] = tok;
      } else {
        asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(tok) : "l"(a.tok_in) : "memory");
      }
      tok = tok < 0 ? 0 : (tok >= a.vocab ? a.vocab - 1 : tok);
      xg = a.embed + (long long)tok * K;
    }
    uint4 xv[XU];
#pragma unroll
    for (int u = 0; u < XU; ++u) {
      const int c = tid + u * CONSUMERS;
      xv[u] = (c < nch) ? ld_cg_v4(xg + c * 8) : make_uint4(0, 0, 0, 0);
    }
    if (a.embed != nullptr && a.h_out != nullptr && blockIdx.x == 0) {
#pragma unroll
      for (int u = 0; u < XU; ++u) {
        const int c = tid + u * CONSUMERS;
        if (c < nch) *reinterpret_cast<uint4*>(a.h_out + c * 8) = xv[u];
      }
    }
    if (a.norm_w != nullptr) {
      float ss = 0.f;
#pragma unroll
      for (int u = 0; u < XU; ++u) {
        const uint4 v = xv[u];
        const float f0 = bf16lo(v.x), f1 = bf16hi(v.x), f2 = bf16lo(v.y), f3 = bf16hi(v.y);
        const float f4 = bf16lo(v.z), f5 = bf16hi(v.z), f6 = bf16lo(v.w), f7 = bf16hi(v.w);
        ss += f0 * f0 + f1 * f1 + f2 * f2 + f3 * f3 + f4 * f4 + f5 * f5 + f6 * f6 + f7 * f7;
      }
      ss = warp_sum(ss);
      if (lane == 0) red[warp] = ss;
      cbar();
      float tot = 0.f;
#pragma unroll
      for (int w = 0; w < CWARPS; ++w) tot += red[w];
      const float rstd = rsqrtf(tot / (float)K + a.eps);
#pragma unroll
      for (int u = 0; u < XU; ++u) {
        const int c = tid + u * CONSUMERS;
        if (c < nch) {
          const uint4 v = xv[u];
          const uint4 gw = *reinterpret_cast<const uint4*>(xs + c * 8);
          uint4 o;
          o.x = bf16x2_mul(gw.x, pack_bf16x2(bf16lo(v.x) * rstd, bf16hi(v.x) * rstd));
          o.y = bf16x2_mul(gw.y, pack_bf16x2(bf16lo(v.y) * rstd, bf16hi(v.y) * rstd));
          o.z = bf16x2_mul(gw.z, pack_bf16x2(bf16lo(v.z) * rstd, bf16hi(v.z) * rstd));
          o.w = bf16x2_mul(gw.w, pack_bf16x2(bf16lo(v.w) * rstd, bf16hi(v.w) * rstd));
          *reinterpret_cast<uint4*>(xs + c * 8) = o;
        }
      }
    } else {
#pragma unroll
      for (int u = 0; u < XU; ++u) {
        const int c = tid + u * CONSUMERS;
        if (c < nch) *reinterpret_cast<uint4*>(xs + c * 8) = xv[u];
      }
    }
  }
  cbar();
  if (tid == 0) trace(2);

  for (int grp = 0; grp < ng; ++grp) {
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    for (int kc = 0; kc < nkc; ++kc) {
      const int kb_n = min(KC, K - kc * KC) >> 5;        // 32-wide K blocks in this slot
      mbar_wait(full_bar(slot), par);
      const uint8_t* base = smem + slot * RG::SLOT;
#pragma unroll
      for (int t = 0; t < KC / 32 / CWARPS; ++t) {
        const int kb = warp + CWARPS * t;
        if (kb < kb_n) {
          uint4 wa, wb;                                                                            // rows g, g+8
          load_a<FMT>(base, kb, lane, wa, wb);
          uint4 xq = make_uint4(0, 0, 0, 0);
          if (g < NB) xq = *reinterpret_cast<const uint4*>(xs + (size_t)g * K + kc * KC + kb * 32 + q * 8);   // column g = clip g
          mma_bf16(c, wa.x, wb.x, wa.y, wb.y, xq.x, xq.y);
          mma_bf16(c, wa.z, wb.z, wa.w, wb.w, xq.z, xq.w);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(slot));
      advance();
    }
    // the 8 per-warp partials of this row group meet in shared memory (double-buffered: the barrier
    // of the next group orders the reads below before the buffer is written again)
    float* pb = pbuf + (grp & 1) * CWARPS * 16 * 4;
    if (q < 2) {                                    // columns (clips) 2q, 2q+1: rows g (c[0], c[1]) and g+8 (c[2], c[3])
      *reinterpret_cast<float2*>(pb + (warp * 16 + g) * 4 + 2 * q) = make_float2(c[0], c[1]);
      *reinterpret_cast<float2*>(pb + (warp * 16 + g + 8) * 4 + 2 * q) = make_float2(c[2], c[3]);
    }
    cbar();
    if (tid < 64) {                                 // (row, clip) = (tid / 4, tid % 4)
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < CWARPS; ++w) v += pb[w * 64 + tid];
      if constexpr (FMT == W_FP8) {
        const int row = row0 + grp * 16 + (tid >> 2);
        if (row < N) v = row_scaled<FMT>(a, row, v);
      }
      result[grp * 64 + tid] = v;
    }
  }
  cbar();
  if (tid == 0) trace(3);

  // ---------------- fused epilogue ----------------
  const bool pairs = (mode == GEMV_SWIGLU || mode == GEMV_QKV);
  const int R = ng * 16;
  const int n_items = (pairs ? R / 2 : R) * NB;     // item = (row or row pair, clip), clip fastest for NB > 1
  for (int it0 = 0; it0 < n_items; it0 += CONSUMERS) {          // uniform trip count: the warps stay converged
    const int it = it0 + tid;
    const int b = (NB == 1) ? 0 : it % NB;
    const int iu = (NB == 1) ? it : it / NB;
    const int rr = pairs ? 2 * iu : iu;
    const int vrow = row0 + rr;
    if (it < n_items && vrow < N) {
      const float v0 = result[rr * 4 + b];
      const float v1 = pairs ? result[(rr + 1) * 4 + b] : 0.f;
      if (mode == GEMV_RES) epi_residual(e, b, vrow, v0);
      else if (mode == GEMV_LOGITS) epi_logit(e, b, vrow, v0);
      else if (mode == GEMV_SWIGLU) epi_swiglu(e, b, vrow, NB, v0, v1);
      else epi_qkv_rope(e, b, vrow, decode_col(e, b), __ldg(e.n_pad + b), v0, v1);
    }
  }
  if (mode == GEMV_LOGITS && a.amax_out != nullptr) {
    // per-CTA partial arg-max over this CTA's rows (bf16-rounded logits, lowest index wins ties);
    // the consumer of the partials keeps the lowest index across CTAs as well
    for (int b = 0; b < NB; ++b) {
      float bv = -INFINITY; int bi = 0x7fffffff;
      for (int rr = tid; rr < R; rr += CONSUMERS) {
        const int vrow = row0 + rr;
        if (vrow < N) {
          const float v = bf16r(result[rr * 4 + b]);
          if (v > bv) { bv = v; bi = vrow; }          // rr ascending: the first maximum is kept
        }
      }
      warp_argmax(bv, bi);
      cbar();                                          // pbuf is free (and the previous clip's slots read)
      if (lane == 0) { pbuf[2 * warp] = bv; pbuf[2 * warp + 1] = __int_as_float(bi); }
      cbar();
      if (tid == 0) {
#pragma unroll
        for (int w = 1; w < CWARPS; ++w) argmax_take(bv, bi, pbuf[2 * w], __float_as_int(pbuf[2 * w + 1]));
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

// ---------------------------------------------------------------------------------------------
// 5..64 clips. NG = upper bound of the row groups a CTA owns (the accumulator arrays are sized and
// unrolled by it), CG = clip groups of 16; a.x holds the activations in the xwin layout
// ---------------------------------------------------------------------------------------------
template <int NG, int CG, int FMT>
__global__ void __launch_bounds__(THREADS, 1) gemv_tcw_kernel(const GemvArgs a, const GemvEpilogue e, const int r0) {
  using RG = Ring<FMT>;
  using P = TwPlan<CG, FMT>;
  constexpr int KP = CWARPS / CG;                     // K phases
  constexpr int TPW = KC / 32 / KP;                   // 32-wide K blocks per warp and slot
  constexpr int TP = 16 * CG + 1;                     // floats per row of a partial tile (padded rows)
  static_assert((P::NWIN & (P::NWIN - 1)) == 0 && P::SMEM <= 227 * 1024, "window area");
  static_assert(KP * NG * 16 * TP * 4 <= P::RING + P::XAREA, "partial tiles");
  extern __shared__ __align__(128) uint8_t smem[];
  // layout: ring[P::NSLOT] | x windows [NWIN][16 CG][1088 B] | barriers; after the main loop the partial tiles
  // [kp][group][16][TP] fp32 take the ring and window memory
  uint8_t* xs = smem + P::RING;
  uint64_t* bars = reinterpret_cast<uint64_t*>(xs + P::XAREA);
  const uint32_t ring0 = smem_u32(smem), xs0 = smem_u32(xs), bar0 = smem_u32(bars);
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (P::NSLOT + s); };
  auto xfull_bar = [&](int s) { return bar0 + 8u * (2 * P::NSLOT + s); };
  auto xempty_bar = [&](int s) { return bar0 + 8u * (2 * P::NSLOT + P::NWIN + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = a.K, N = a.N, NB = a.B;
  const int nkc = (K + KC - 1) / KC;
  int grp_begin;
  const int ng = cta_row_groups(N, grp_begin);        // 1..NG

  if (tid == 0) {
    for (int s = 0; s < P::NSLOT; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), CWARPS); }
    for (int s = 0; s < P::NWIN; ++s) { mbar_init(xfull_bar(s), 1); mbar_init(xempty_bar(s), CWARPS); }
    mbar_fence_init();
  }
  // rows of the activation windows that no clip owns stay zero (their MMA columns are never stored)
  for (int i = tid; i < P::XAREA / 16; i += THREADS) reinterpret_cast<uint4*>(xs)[i] = make_uint4(0, 0, 0, 0);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  pdl_launch_dependents();

  if (warp == CWARPS) {
    // =============================== producer ===============================
    // (32-bit index arithmetic only: a 64-bit division here becomes a subroutine call inside the
    // single-lane region and the uniform-datapath code around the bulk copies then faults)
    if (lane == 0) {
      const int total = ng * nkc;
      const int pre = total < P::NSLOT ? total : P::NSLOT;
      const uint8_t* W = weight_bytes<FMT>(a);
      // the weights never depend on the previous kernel: fill the ring before the dependency wait
      {
        int kc = 0, lg = 0;
        for (int idx = 0; idx < pre; ++idx) {
          const uint32_t bytes = (uint32_t)min(KC, K - kc * KC) * (16u * RG::EB);
          const uint8_t* src = W + ((size_t)(grp_begin + lg) * 16 * K + (size_t)kc * KC * 16) * RG::EB;
          mbar_arrive_expect_tx(full_bar(idx), bytes);
          bulk_g2s(ring0 + idx * RG::SLOT, src, bytes, full_bar(idx));
          if (++lg == ng) { lg = 0; ++kc; }
        }
      }
      pdl_wait();
      int idx = 0, slot = 0, use = 0;                 // slot = idx % NSLOT, use = idx / NSLOT
      const uint32_t win_bytes = (uint32_t)NB * TW_XROW;
      for (int kc = 0; kc < nkc; ++kc) {
        const int xb = kc & (P::NWIN - 1);
        if (kc >= P::NWIN) mbar_wait(xempty_bar(xb), (uint32_t)(((kc / P::NWIN) - 1) & 1));
        mbar_arrive_expect_tx(xfull_bar(xb), win_bytes);
        bulk_g2s(xs0 + xb * P::XBUF, a.x + (size_t)kc * NB * XWIN_PITCH, win_bytes, xfull_bar(xb));
        for (int lg = 0; lg < ng; ++lg) {
          if (idx >= pre) {
            const uint32_t bytes = (uint32_t)min(KC, K - kc * KC) * (16u * RG::EB);
            const uint8_t* src = W + ((size_t)(grp_begin + lg) * 16 * K + (size_t)kc * KC * 16) * RG::EB;
            mbar_wait(empty_bar(slot), (uint32_t)((use - 1) & 1));
            mbar_arrive_expect_tx(full_bar(slot), bytes);
            bulk_g2s(ring0 + slot * RG::SLOT, src, bytes, full_bar(slot));
          }
          ++idx;
          if (++slot == P::NSLOT) { slot = 0; ++use; }
        }
      }
    }
    return;
  }

  // =============================== consumers ===============================
  pdl_wait();                                           // the epilogue reads / overwrites tensors of earlier kernels
  const int g = lane >> 2, q = lane & 3;
  // K phase and clip group of this warp (the compiler cannot prove warp < 8 here: CG = 1 spells out kp = warp)
  const int kp = CG == 1 ? warp : warp % KP, cg = CG == 1 ? 0 : warp / KP;
  float acc[NG][2][4];
#pragma unroll
  for (int i = 0; i < NG; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

  int slot = 0;
  uint32_t par = 0;
  for (int kc = 0; kc < nkc; ++kc) {
    const int xb = kc & (P::NWIN - 1);
    const int kb_n = min(KC, K - kc * KC) >> 5;          // 32-wide K blocks in this chunk
    mbar_wait(xfull_bar(xb), (uint32_t)((kc / P::NWIN) & 1));
    const uint8_t* xw = xs + xb * P::XBUF;
    // this warp's share of every slot of the chunk: K blocks kp, kp + KP, ...; the B fragments (the activations
    // of its 16 clips for those K blocks) are the same for every row group: load them once
    uint4 xq[TPW][2];
#pragma unroll
    for (int t = 0; t < TPW; ++t)
#pragma unroll
      for (int j = 0; j < 2; ++j)
        xq[t][j] = *reinterpret_cast<const uint4*>(xw + (16 * cg + 8 * j + g) * TW_XROW + (kp + KP * t) * 64 + q * 16);
#pragma unroll
    for (int i = 0; i < NG; ++i) {
      if (i < ng) {
        mbar_wait(full_bar(slot), par);
        const uint8_t* base = smem + slot * RG::SLOT;
#pragma unroll
        for (int t = 0; t < TPW; ++t) {
          const int kb = kp + KP * t;
          if (kb < kb_n) {
            uint4 wa, wb;                                                                              // rows g, g + 8
            load_a<FMT>(base, kb, lane, wa, wb);
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              mma_bf16(acc[i][j], wa.x, wb.x, wa.y, wb.y, xq[t][j].x, xq[t][j].y);
              mma_bf16(acc[i][j], wa.z, wb.z, wa.w, wb.w, xq[t][j].z, xq[t][j].w);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(slot));
        if (++slot == P::NSLOT) { slot = 0; par ^= 1u; }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(xempty_bar(xb));
  }

  // ---------------- the KP partial tiles of every group and clip meet in the (now idle) shared memory ----------------
  cbar();                                               // every warp has left the ring and the windows
  float* tiles = reinterpret_cast<float*>(smem);        // [kp][group][16][TP]
#pragma unroll
  for (int i = 0; i < NG; ++i) {
    if (i < ng) {
      float* t = tiles + ((size_t)kp * NG + i) * 16 * TP + 16 * cg;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        t[g * TP + 8 * j + 2 * q] = acc[i][j][0];
        t[g * TP + 8 * j + 2 * q + 1] = acc[i][j][1];
        t[(g + 8) * TP + 8 * j + 2 * q] = acc[i][j][2];
        t[(g + 8) * TP + 8 * j + 2 * q + 1] = acc[i][j][3];
      }
    }
  }
  cbar();

  // ---------------- fused epilogue ----------------
  // All 256 consumer threads share the items of every group, one pass per clip group: thread = (row or row pair,
  // clip) with the ROW index fastest, so that a warp's accesses to the residual / output rows are contiguous runs
  // (a warp per group walking (row, clip) items with the clip fastest touched 32 sectors per instruction, one
  // dependent round trip per 32 items at the end of every launch). The KP partial tiles are summed on the fly,
  // in a fixed order.
  const int mode = e.mode;
  const bool pairs = (mode == GEMV_SWIGLU || mode == GEMV_QKV);
  auto tile_sum = [&](int lg, int el) {
    float v = tiles[(size_t)lg * 16 * TP + el];
#pragma unroll
    for (int k2 = 1; k2 < KP; ++k2) v += tiles[((size_t)k2 * NG + lg) * 16 * TP + el];
    return v;
  };
  if (!pairs) {
    const int rr = tid & 15;                             // 16 rows x 16 clips of one group per pass
    for (int bb = 0; bb < CG; ++bb) {
      const int b = 16 * bb + (tid >> 4);
#pragma unroll 2
      for (int lg = 0; lg < ng; ++lg) {
        const int vrow = (grp_begin + lg) * 16 + rr;
        if (b < NB && vrow < N) {
          const float v0 = row_scaled<FMT>(a, vrow, tile_sum(lg, rr * TP + b));
          if (mode == GEMV_RES) epi_residual(e, b, r0 + vrow, v0);
          else epi_logit(e, b, r0 + vrow, v0);
        }
      }
    }
  } else {
    const int pr = tid & 7;                              // 8 row pairs x 16 clips of TWO groups per pass
    for (int bb = 0; bb < CG; ++bb) {
      const int b = 16 * bb + ((tid >> 3) & 15);
      int col = 0, floor = 0;                            // q|k|v: clip b's column and key floor, loaded once
      if (mode == GEMV_QKV && b < NB) { col = decode_col(e, b); floor = __ldg(e.n_pad + b); }
      for (int lg = tid >> 7; lg < ng; lg += 2) {
        const int rr = 2 * pr;
        const int vrow = (grp_begin + lg) * 16 + rr;
        if (b >= NB || vrow >= N) continue;
        const float v0 = row_scaled<FMT>(a, vrow, tile_sum(lg, rr * TP + b));
        const float v1 = row_scaled<FMT>(a, vrow + 1, tile_sum(lg, (rr + 1) * TP + b));
        if (mode == GEMV_SWIGLU) epi_swiglu(e, b, r0 + vrow, NB, v0, v1);
        else epi_qkv_rope(e, b, r0 + vrow, col, floor, v0, v1);
      }
    }
  }
}

// row-major W[N][K] -> tiled copy. One thread per 16-byte chunk of the output.
__global__ void gemv_tc_repack_kernel(const bf16* __restrict__ W, bf16* __restrict__ dst, int N, int K, int qkv) {
  const size_t chunks_per_group = (size_t)2 * K;                      // 16 rows x K x 2 B / 16 B
  const size_t n_chunks = (size_t)((N + 15) >> 4) * chunks_per_group;
  for (size_t o = (size_t)blockIdx.x * blockDim.x + threadIdx.x; o < n_chunks; o += (size_t)gridDim.x * blockDim.x) {
    const int grp = (int)(o / chunks_per_group);
    const size_t off = (o - (size_t)grp * chunks_per_group) * 16;     // byte offset inside the group
    const int kc = (int)(off / ((size_t)KC * 32));
    const int within = (int)(off - (size_t)kc * KC * 32);
    const int kb = within >> 10, r = within & 1023;
    const int half = r >> 9, l = (r & 511) >> 4;
    const int row = grp * 16 + (l >> 2) + 8 * half;
    const int k = kc * KC + kb * 32 + (l & 3) * 8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row < N) {
      const long long src_row = qkv ? qkv_row(row) : (long long)row;
      v = *reinterpret_cast<const uint4*>(W + src_row * K + k);
    }
    *reinterpret_cast<uint4*>(dst + o * 8) = v;
  }
}

// Load-time E4M3 quantizer, one CTA per row v of the decode copy (source row qkv_row(v) of a q|k|v matrix, row v
// otherwise). With a = max |W[r, :]|, e is the smallest integer with a <= 448 * 2^e (0 for an all-zero row), so
// the row maximum lands in (224, 448]; q = E4M3(W * 2^-e), round to nearest even with subnormals (exact scaling,
// never above 448: torch's .to(torch.float8_e4m3fn)); W~ = q * 2^e, exactly a bf16. Writes the codes in the slot
// order of the ring kernels (the element order of gemv_tc_repack_kernel, one byte each), scales[v] = 2^e, and W~
// into w_deq[source row] (w_deq may be W: each element is read and then written by one thread). bad (optional):
// bad[0] = the lowest source row with a non-finite weight, bad[1] = the lowest whose 2^e is not a normal fp32
// number or whose W~ is not exactly a finite bf16; rows that pass leave them alone.
__global__ void __launch_bounds__(256) gemv_quantize_fp8_kernel(const bf16* W, bf16* w_deq, uint8_t* __restrict__ codes,
                                                                 float* __restrict__ scales, int N, int K, int qkv,
                                                                 int* bad) {
  __shared__ float red[8];
  const int v = blockIdx.x, tid = threadIdx.x;
  const long long sr = qkv ? qkv_row(v) : (long long)v;
  const bf16* src = W + sr * K;
  const int nch = K >> 3;
  float amax = 0.f;
  bool finite = true;
  for (int c = tid; c < nch; c += 256) {
    const uint4 u = *reinterpret_cast<const uint4*>(src + c * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float f0 = bf16lo(w[i]), f1 = bf16hi(w[i]);
      finite = finite && isfinite(f0) && isfinite(f1);
      amax = fmaxf(amax, fmaxf(fabsf(f0), fabsf(f1)));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((tid & 31) == 0) red[tid >> 5] = amax;
  finite = __syncthreads_and(finite);
  amax = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) amax = fmaxf(amax, red[w]);
  int e = 0;
  if (amax > 0.f) {
    int x;
    const float m = frexpf(amax, &x);                  // amax = m * 2^x, 0.5 <= m < 1; 448 = 0.875 * 2^9
    e = m <= 0.875f ? x - 9 : x - 8;
  }
  const bool e_ok = e >= -126 && e <= 126;
  const int ec = e_ok ? e : 0;
  const float s = __int_as_float((ec + 127) << 23), s_inv = __int_as_float((127 - ec) << 23);
  bool exact = e_ok;
  uint8_t* cg = codes + (size_t)(v >> 4) * 16 * K;     // this row's 16-row group
  const int r = v & 15, half = r >> 3, g = r & 7;
  for (int c = tid; c < nch; c += 256) {
    const uint4 u = *reinterpret_cast<const uint4*>(src + c * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t q[2] = {0u, 0u}, d[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float f[2] = {bf16lo(w[i]), bf16hi(w[i])};
      float wt[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const __nv_fp8_storage_t c8 = __nv_cvt_float_to_fp8(f[j] * s_inv, __NV_SATFINITE, __NV_E4M3);
        q[i >> 1] |= (uint32_t)c8 << (8 * (2 * (i & 1) + j));
        wt[j] = __half2float(__half(__nv_cvt_fp8_to_halfraw(c8, __NV_E4M3))) * s;
      }
      d[i] = pack_bf16x2(wt[0], wt[1]);
      exact = exact && bf16lo(d[i]) == wt[0] && bf16hi(d[i]) == wt[1] && isfinite(wt[0]) && isfinite(wt[1]);
    }
    *reinterpret_cast<uint4*>(w_deq + sr * K + c * 8) = make_uint4(d[0], d[1], d[2], d[3]);
    // k = 8c: K chunk kc, 32-wide block kb, lane (g, k / 8 % 4)
    const int k = c * 8, kc = k / KC, kin = k % KC;
    const size_t off = (size_t)kc * KC * 16 + (kin >> 5) * 512 + half * 256 + (g * 4 + ((kin >> 3) & 3)) * 8;
    *reinterpret_cast<uint2*>(cg + off) = make_uint2(q[0], q[1]);
  }
  exact = __syncthreads_and(exact);
  if (tid == 0) {
    scales[v] = s;
    if (bad != nullptr && !finite) atomicMin(bad, (int)sr);
    if (bad != nullptr && finite && !exact) atomicMin(bad + 1, (int)sr);
  }
}

// ---------------------------------------------------------------------------------------------
// launch layer
// ---------------------------------------------------------------------------------------------
// gemv_tc shared-memory plan on `grid` CTAs; returns the slot count (0 = does not fit). fp8 weights: slots of
// half the size, up to twice as many
int plan(int nb, int N, int K, bool norm, int grid, size_t* smem_bytes, int* x_elems, int* r_cap, int fmt = W_BF16) {
  if (K % 32 != 0 || K > 14336) return 0;
  const int slot_bytes = fmt == W_FP8 ? Ring<W_FP8>::SLOT : SLOT_BYTES;
  const int max_slots = fmt == W_FP8 ? Ring<W_FP8>::NSLOT : SLOTS;
  const int xe = K * (nb + ((nb > 1 && norm) ? 1 : 0));   // x buffer: nb vectors (+ the parked norm weights when nb > 1)
  const int rmax = (((N + 15) / 16 + grid - 1) / grid) * 16;
  const size_t fixed = (size_t)xe * 2 + (size_t)(2 * CWARPS * 16 + rmax) * 4 * 4 + 4 * CWARPS * 4 + 2 * max_slots * 8 + 128;
  const size_t limit = nb > 1 ? TC_SMEM_CLIPS : TC_SMEM_ONE_CLIP;
  if (fixed + 4 * (size_t)slot_bytes > limit) return 0;
  int slots = (int)((limit - fixed) / slot_bytes);
  if (slots > max_slots) slots = max_slots;
  *smem_bytes = (size_t)slots * slot_bytes + fixed;
  *x_elems = xe; *r_cap = rmax;
  return slots;
}

cudaLaunchConfig_t pdl_config(int grid, size_t smem, cudaStream_t stream, cudaLaunchAttribute* attr) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cfg;
}

// VCL_TC_TRACE: every gemv_tc launch writes 8 timestamps per CTA into the next record of a device buffer;
// vcl_debug_tc_trace_dump() (below) writes the records to a file. Debug aid for eager runs.
constexpr int TC_TRACE_RECORDS = 512;
unsigned long long* g_trace = nullptr;
int g_trace_next = 0;

// the weights of a launch: the bf16 slots or the fp8 codes (with their row scales), 16-byte aligned
int weight_format(const GemvArgs& a) {
  VCL_REQUIRE((a.W_tiled != nullptr) != (a.W_fp8 != nullptr) && (a.W_fp8 == nullptr) == (a.w_scale == nullptr),
              "gemv: exactly one of the bf16 copy (W_tiled) or the fp8 codes with their row scales (W_fp8, w_scale)");
  VCL_REQUIRE((uintptr_t)a.W_tiled % 16 == 0 && (uintptr_t)a.W_fp8 % 16 == 0, "gemv: weights must be 16-byte aligned");
  return a.W_fp8 != nullptr ? W_FP8 : W_BF16;
}

int launch_tc(const GemvArgs& a, const GemvEpilogue& e, cudaStream_t stream) {
  VCL_REQUIRE(!e.out_xwin, "gemv: the 1..4-clip kernel writes row-major outputs only (out_xwin)");
  VCL_REQUIRE(a.ldx % 8 == 0 && (a.embed != nullptr || (uintptr_t)a.x % 16 == 0),
              "gemv_tc: operands must be 16-byte aligned");
  const int fmt = weight_format(a);
  if (fmt < 0) return fmt;
  TcParams p = {};
  p.a = a; p.e = e;
  const int grid = gemv_grid(a.N);
  size_t smem = 0;
  p.n_slots = plan(a.B, a.N, a.K, a.norm_w != nullptr, grid, &smem, &p.x_elems, &p.r_cap, fmt);
  VCL_REQUIRE(p.n_slots >= 4, "gemv_tc: B=%d N=%d K=%d does not fit the shared-memory plan", a.B, a.N, a.K);
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
  cudaLaunchAttribute attr[1];
  cudaLaunchConfig_t cfg = pdl_config(grid, smem, stream, attr);
  VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, fmt == W_FP8 ? gemv_tc_kernel<W_FP8> : gemv_tc_kernel<W_BF16>, p));
  count_launches(1);
  return 0;
}

typedef void (*TcwKernel)(const GemvArgs, const GemvEpilogue, const int);
struct TcwInstance { TcwKernel kern; int ng, smem; };
template <int NG, int CG, int FMT> TcwInstance tcw() { return {gemv_tcw_kernel<NG, CG, FMT>, NG, TwPlan<CG, FMT>::SMEM}; }
// [format][CG = 1, 2, 4][instance], NG ascending (unused entries: ng = 0); the largest NG of a CG is the largest
// instance without spills
const TcwInstance tcw_kernels[2][3][4] = {
    {{tcw<2, 1, W_BF16>(), tcw<6, 1, W_BF16>(), tcw<10, 1, W_BF16>(), tcw<14, 1, W_BF16>()},
     {tcw<2, 2, W_BF16>(), tcw<6, 2, W_BF16>(), tcw<10, 2, W_BF16>()},
     {tcw<2, 4, W_BF16>(), tcw<4, 4, W_BF16>(), tcw<6, 4, W_BF16>()}},
    {{tcw<2, 1, W_FP8>(), tcw<6, 1, W_FP8>(), tcw<10, 1, W_FP8>(), tcw<14, 1, W_FP8>()},
     {tcw<2, 2, W_FP8>(), tcw<6, 2, W_FP8>(), tcw<10, 2, W_FP8>()},
     {tcw<2, 4, W_FP8>(), tcw<4, 4, W_FP8>(), tcw<6, 4, W_FP8>()}}};

// 5..64 clips: a matrix with more row groups per SM than the largest instance of its CG takes runs as consecutive
// launches over near-equal row slices; the epilogue addresses rows by their index in the whole matrix
int launch_tcw(const GemvArgs& a, const GemvEpilogue& e, cudaStream_t stream) {
  VCL_REQUIRE(a.norm_w == nullptr && a.embed == nullptr && a.amax_out == nullptr,
              "gemv: the 5..64-clip kernel takes normalised activations (no fused norm, embedding gather or "
              "arg-max partials)");
  VCL_REQUIRE((uintptr_t)a.x % 16 == 0, "gemv_tcw: operands must be 16-byte aligned");
  const int fmt = weight_format(a);
  if (fmt < 0) return fmt;
  const TcwInstance* inst = tcw_kernels[fmt][a.B <= 16 ? 0 : a.B <= 32 ? 1 : 2];   // 1, 2 or 4 clip groups of 16
  int ng_cap = 0;
  for (int i = 0; i < 4; ++i) ng_cap = inst[i].ng > ng_cap ? inst[i].ng : ng_cap;
  const int groups = (a.N + 15) / 16, sms = device_num_sms();
  const int n_slices = (groups + ng_cap * sms - 1) / (ng_cap * sms);
  for (int s = 0; s < n_slices; ++s) {
    const int g0 = (int)((long long)groups * s / n_slices), g1 = (int)((long long)groups * (s + 1) / n_slices);
    const long long r0 = (long long)g0 * 16;
    GemvArgs sa = a;
    if (fmt == W_FP8) {
      sa.W_fp8 = a.W_fp8 + r0 * a.K;
      sa.w_scale = a.w_scale + r0;
    } else {
      sa.W_tiled = a.W_tiled + r0 * a.K;
    }
    sa.N = (a.N < g1 * 16 ? a.N : g1 * 16) - (int)r0;
    const int grid = g1 - g0 < sms ? g1 - g0 : sms;                   // no CTA without a row group
    const int ng_max = (g1 - g0 + grid - 1) / grid;                  // groups of the busiest CTA
    int pick = 0;
    while (inst[pick].ng < ng_max) ++pick;
    cudaLaunchAttribute attr[1];
    cudaLaunchConfig_t cfg = pdl_config(grid, inst[pick].smem, stream, attr);
    VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, inst[pick].kern, sa, e, (int)r0));
    count_launches(1);
  }
  return 0;
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

int init_gemv_kernels() {
  for (auto k : {gemv_tc_kernel<W_BF16>, gemv_tc_kernel<W_FP8>})
    VCL_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024));
  for (const auto& by_fmt : tcw_kernels)
    for (const auto& by_cg : by_fmt)
      for (const TcwInstance& k : by_cg)
        if (k.kern != nullptr) VCL_CUDA_OK(cudaFuncSetAttribute(k.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, k.smem));
  return 0;
}

// one CTA per SM, but none without a row group
int gemv_grid(int N) {
  const int n_groups = (N + 15) / 16, sms = device_num_sms();
  return n_groups < sms ? n_groups : sms;
}

bool gemv_fits(int B, int N, int K, bool norm, bool fp8) {
  if (B < 1 || B > 64 || N < 1) return false;
  if (B > 4) return K % 32 == 0;              // 5..64 clips: any matrix, in row slices
  size_t smem = 0; int xe = 0, rc = 0;
  return plan(B, N, K, norm, gemv_grid(N), &smem, &xe, &rc, fp8 ? W_FP8 : W_BF16) >= 4;
}

size_t gemv_tiled_elems(int N, int K) { return (size_t)((N + 15) / 16) * 16 * K; }

int launch_gemv_repack(const bf16* W, bf16* dst, int N, int K, bool qkv_pairs, cudaStream_t stream) {
  VCL_REQUIRE(K % 32 == 0, "gemv repack: K=%d must be a multiple of 32", K);
  VCL_REQUIRE(!qkv_pairs || N % 128 == 0, "gemv repack: q/k/v rows must come in heads of 128 (N=%d)", N);
  gemv_tc_repack_kernel<<<device_num_sms() * 8, 256, 0, stream>>>(W, dst, N, K, qkv_pairs ? 1 : 0);
  VCL_CUDA_OK(cudaGetLastError());
  return 0;
}

int launch_gemv_quantize_fp8(const bf16* W, bf16* w_deq, uint8_t* codes, float* scales, int N, int K, bool qkv_pairs,
                             int* bad, cudaStream_t stream) {
  VCL_REQUIRE(N >= 1 && K >= 32 && K % 32 == 0, "fp8 quantizer: N=%d K=%d (K a positive multiple of 32)", N, K);
  VCL_REQUIRE(!qkv_pairs || N % 128 == 0, "fp8 quantizer: q/k/v rows must come in heads of 128 (N=%d)", N);
  VCL_REQUIRE((uintptr_t)W % 16 == 0 && (uintptr_t)w_deq % 16 == 0 && (uintptr_t)codes % 16 == 0,
              "fp8 quantizer: operands must be 16-byte aligned");
  // the rows of the last 16-row group past N stay zero
  VCL_CUDA_OK(cudaMemsetAsync(codes, 0, gemv_tiled_elems(N, K), stream));
  gemv_quantize_fp8_kernel<<<N, 256, 0, stream>>>(W, w_deq, codes, scales, N, K, qkv_pairs ? 1 : 0, bad);
  VCL_CUDA_OK(cudaGetLastError());
  return 0;
}

int launch_gemv(const GemvArgs& a, const GemvEpilogue& e, cudaStream_t stream) {
  VCL_REQUIRE(e.mode >= GEMV_RES && e.mode <= GEMV_LOGITS, "gemv: unknown epilogue mode %d", e.mode);
  VCL_REQUIRE(gemv_fits(a.B, a.N, a.K, a.norm_w != nullptr, a.W_fp8 != nullptr),
              "gemv: B=%d N=%d K=%d is outside the decode kernels' range (1..64 clips, K a multiple of 32; "
              "1..4 clips: K <= 14336 and the shared-memory plan)", a.B, a.N, a.K);
  VCL_REQUIRE(e.mode != GEMV_SWIGLU || a.N % 2 == 0, "gemv swiglu: N must be even (interleaved gate/up rows)");
  VCL_REQUIRE(e.mode != GEMV_QKV || a.N == 3 * e.H * 128, "gemv qkv: N=%d != 3*H*128", a.N);
  VCL_REQUIRE((e.n_pad != nullptr) == (e.mode == GEMV_QKV),
              "gemv: the q|k|v epilogue needs the key floors n_pad, and no other epilogue takes them");
  VCL_REQUIRE(a.embed == nullptr || (a.vocab > 0 && (a.tok_in != nullptr || (a.amax_in != nullptr && a.amax_n > 0))),
              "gemv: the fused embedding gather needs a token source");
  return a.B <= 4 ? launch_tc(a, e, stream) : launch_tcw(a, e, stream);
}

}  // namespace vcl

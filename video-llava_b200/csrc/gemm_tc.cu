// Dense bf16 GEMM on the Hopper warpgroup tensor cores:  C[M,N] = epilogue(A[M,K] . W[N,K]^T)
//
// This one kernel serves every dense contraction on the hot path (SURVEY.md section 2.3 rows
// V1, V3, V5-V7, J1, L1, L4-L6): both operands are K-major exactly as nn.Linear stores them
// (activations [rows, K], weights [out, in]), so no transposes are ever materialised.
//
//   warpgroup 0, warp 0, lane 0  TMA producer : issues cp.async.bulk.tensor 2-D tiles (128B swizzle) into a
//                                               smem ring; the warpgroup hands most of its registers to the
//                                               consumers
//   warpgroup 0, warps 1-3       store warps  : read each staged 64-row block back as 16-byte row chunks
//                                               (+ residual) and store whole contiguous row segments per
//                                               instruction, while the consumers run the next tile
//   warpgroups 1-2               consumers    : 64 rows each of the 128 x BLOCK_N tile, wgmma.mma_async
//                                               m64nBLOCK_Nk16 with fp32 accumulators in registers; the stage is
//                                               released once the wgmma that read it has retired (one group kept
//                                               in flight); then accumulators -> bias / activation / RoPE -> bf16
//                                               into their padded staging block in shared memory
//
// Persistent: grid = the number of CTAs (clusters) that fit at once, capped by the tile count; the producer
// runs ahead into the next tile while the consumers stage the current one, and the store warps drain a staged
// block while the consumers' tensor cores work on the next tile (one staging block per consumer warpgroup,
// handed over through the staged / drained mbarriers).
//
// Rounding points reproduce the reference's eager bf16 path (each nn.Linear output is rounded to
// bf16 before the following elementwise op):
//   CLIP quick_gelu  x*sigmoid(1.702x)   transformers/activations.py:117-123
//   CLIP residual    hidden + out        transformers/models/clip/modeling_clip.py:377,382
//   LLaMA SwiGLU     silu(gate)*up       transformers/models/llama/modeling_llama.py:182-184
//   LLaMA residual                       transformers/models/llama/modeling_llama.py:325,331
//   LLaMA RoPE + KV-cache write (ACT_ROPE, the prefill's q|k|v projection)
//                                        transformers/models/llama/modeling_llama.py:124-168
#include "common.cuh"
#include "kernels.h"

#include <cudaTypedefs.h>

namespace vcl {

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int BLOCK_M = 128;
  static constexpr int BLOCK_K = 64;  // 64 bf16 = one 128-byte swizzle span
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int OUT_PITCH = BLOCK_N * 2 + 16;     // bytes per staged output row (+16: no bank conflicts)
  static constexpr int OUT_BYTES = BLOCK_M * OUT_PITCH;
  static constexpr int BAR_BYTES = 256;
  // as many ring stages as fit next to the staging block in the 227 KB a CTA may use
  static constexpr int STAGES = (BLOCK_N == 256) ? 3 : (BLOCK_N == 128 ? 5 : 8);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + OUT_BYTES + 1024;  // +1024: manual align
  static_assert((2 * STAGES + 4) * 8 <= BAR_BYTES, "barrier area");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
};

__device__ __forceinline__ float act_gelu_erf(float x) {
  x = bf16r(x);
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
}

// Epilogue, phase 1: this warpgroup's 64 x BLOCK_N accumulators -> bf16 outputs in the staging block
// (stg = its first row). Each thread holds column pairs (2c, 2c+1) of two rows (accumulator layout in common.cuh).
//   ACT_SWIGLU: weight rows are interleaved (2j = gate_j, 2j+1 = up_j), so a pair is one output column j.
//   ACT_ROPE  : a 128-column block is one head of q | k | v; the RoPE partner of column d is d + 64, which the
//               same thread holds 8 accumulator groups further on, so the rotation is thread-local. Arithmetic =
//               rope_kv_prefill_kernel (elementwise.cu): x rounded to bf16, every product rounded, fp32 sum, one
//               final rounding (transformers/models/llama/modeling_llama.py:124-168). With left padding
//               (rp.n_pad) the angle is that of cache column - n_pad[clip], clamped at 0; the columns do not move.
//               Packed rows (rp.pack): the angle is the row's position in its sequence.
template <int BLOCK_N, int ACT>
__device__ __forceinline__ void gemm_epilogue_stage(const float (&acc)[BLOCK_N / 2], uint8_t* stg, int lane, int wq,
                                                    int row_base, int n_blk, const bf16* __restrict__ bias, int M,
                                                    int N, const RopeEpilogue& rp) {
  using Cfg = GemmCfg<BLOCK_N>;
  const int r0 = 16 * wq + (lane >> 2);
  const int c2 = 2 * (lane & 3);
  if constexpr (ACT == ACT_ROPE) {
    static_assert(BLOCK_N % 128 == 0, "one head (128 columns) per tile at least");
#pragma unroll
    for (int hh = 0; hh < BLOCK_N / 128; ++hh) {
      const int gh = n_blk * (BLOCK_N / 128) + hh;               // head index over q | k | v
      const int which = gh / rp.H;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        const int grow = row_base + r;
        int pos;
        if (rp.pack != nullptr) {
          pos = grow < M ? __ldg(pack_row(rp.pack, grow) + 1) : 0;                                  // packed rows
        } else {
          pos = rp.start_pos + (grow < M ? grow % rp.S : 0);
          if (rp.n_pad != nullptr && grow < M) pos = max(pos - __ldg(rp.n_pad + grow / rp.S), 0);   // left padding
        }
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = hh * 16 + jj, d = 8 * jj + c2;
          const uint32_t l2 = pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          const uint32_t h2 = pack_bf16x2(acc[4 * (j + 8) + 2 * h], acc[4 * (j + 8) + 2 * h + 1]);
          uint32_t olo = l2, ohi = h2;
          if (which != 2 && grow < M) {
            const uint32_t cw = __ldg(reinterpret_cast<const uint32_t*>(rp.cos_t + (long long)pos * 64 + d));
            const uint32_t sw = __ldg(reinterpret_cast<const uint32_t*>(rp.sin_t + (long long)pos * 64 + d));
            const float l0 = bf16lo(l2), l1 = bf16hi(l2), h0 = bf16lo(h2), h1 = bf16hi(h2);
            const float c0 = bf16lo(cw), c1 = bf16hi(cw), s0 = bf16lo(sw), s1 = bf16hi(sw);
            olo = pack_bf16x2(bf16r(l0 * c0) + bf16r(-h0 * s0), bf16r(l1 * c1) + bf16r(-h1 * s1));
            ohi = pack_bf16x2(bf16r(h0 * c0) + bf16r(l0 * s0), bf16r(h1 * c1) + bf16r(l1 * s1));
          }
          *reinterpret_cast<uint32_t*>(stg + r * Cfg::OUT_PITCH + (hh * 128 + d) * 2) = olo;
          *reinterpret_cast<uint32_t*>(stg + r * Cfg::OUT_PITCH + (hh * 128 + 64 + d) * 2) = ohi;
        }
      }
    }
  } else {
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int col = 8 * j + c2;
      const int gcol = n_blk * BLOCK_N + col;
      float b0 = 0.f, b1 = 0.f;
      if (bias != nullptr && gcol < N) {
        const uint32_t bw = __ldg(reinterpret_cast<const uint32_t*>(bias + gcol));
        b0 = bf16lo(bw); b1 = bf16hi(bw);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        const float x0 = acc[4 * j + 2 * h] + b0, x1 = acc[4 * j + 2 * h + 1] + b1;
        if constexpr (ACT == ACT_SWIGLU) {
          const float g = bf16r(x0);
          const bf16 s = __float2bfloat16_rn(act_sigmoid_div(g, g));                  // silu (bf16)
          const bf16 o = __hmul(s, __float2bfloat16_rn(x1));                           // * up (bf16)
          *reinterpret_cast<bf16*>(stg + r * Cfg::OUT_PITCH + col) = o;                // output column col / 2
        } else {
          uint32_t o;
          if constexpr (ACT == ACT_QGELU) {
            // x*sigmoid(1.702x): the three bf16 tensors of the reference are materialised
            const uint32_t x2 = pack_bf16x2(x0, x1);
            const uint32_t t2 = pack_bf16x2(1.702f * bf16lo(x2), 1.702f * bf16hi(x2));
            const uint32_t s2 = pack_bf16x2(act_sigmoid_div(1.0f, bf16lo(t2)), act_sigmoid_div(1.0f, bf16hi(t2)));
            o = bf16x2_mul(x2, s2);
          } else if constexpr (ACT == ACT_GELU) {
            o = pack_bf16x2(act_gelu_erf(x0), act_gelu_erf(x1));
          } else {
            o = pack_bf16x2(x0, x1);
          }
          *reinterpret_cast<uint32_t*>(stg + r * Cfg::OUT_PITCH + col * 2) = o;
        }
      }
    }
  }
}

// Epilogue, phase 2 (the store warps): the staged 64-row block leaves as 16-byte chunks, consecutive threads on
// consecutive chunks of a row (whole contiguous row segments per store instruction); the residual is added here,
// one more bf16 rounding (packed bf16x2 add). ACT_ROPE: q goes to C, k and v straight into the KV cache.
// The store warps have a whole mainloop to drain a block; the residual GEMMs need 64 KB in per 128 x 256 tile,
// so each thread first issues RES_INFLIGHT residual loads and only then adds and stores them. 96 is a multiple of
// every chunk count per row (4 ... 32), so a store thread keeps one column chunk and walks down the rows.
constexpr int STORE_THREADS = 96;     // warps 1-3 of warpgroup 0
constexpr int RES_INFLIGHT = 4;       // 16-byte residual loads in flight per store thread
template <int BLOCK_N, int ACT>
__device__ __forceinline__ void gemm_epilogue_store(const uint8_t* stg, int t, int row_base, int n_blk, bf16* C,
                                                    long long ldc, const bf16* residual, long long ldr, int M, int N,
                                                    const RopeEpilogue& rp) {
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int OUT_W = ACT == ACT_SWIGLU ? BLOCK_N / 2 : BLOCK_N;
  constexpr int CPR = OUT_W / 8;                      // 16-byte chunks per row
  constexpr int RSTEP = STORE_THREADS / CPR;          // rows between a thread's consecutive chunks
  static_assert(STORE_THREADS % CPR == 0, "one column chunk per store thread");
  constexpr bool RES = ACT != ACT_ROPE && ACT != ACT_SWIGLU;
  const int n_out = ACT == ACT_SWIGLU ? N / 2 : N;
  const int c = t % CPR, col = n_blk * OUT_W + c * 8;
  if (col >= n_out) return;
  const int rows = min(64, M - row_base);
  for (int r0 = t / CPR; r0 < rows; r0 += RSTEP * RES_INFLIGHT) {
    uint4 rr[RES_INFLIGHT];
    if (RES && residual != nullptr) {
#pragma unroll
      for (int u = 0; u < RES_INFLIGHT; ++u) {
        const int r = r0 + u * RSTEP;
        if (r < rows) rr[u] = *reinterpret_cast<const uint4*>(residual + (long long)(row_base + r) * ldr + col);
      }
    }
    // ACT_ROPE: not unrolled, the cache address of a row (a map lookup for packed rows) fits the store warps'
    // registers one row at a time
#pragma unroll (ACT == ACT_ROPE ? 1 : RES_INFLIGHT)
    for (int u = 0; u < RES_INFLIGHT; ++u) {
      const int r = r0 + u * RSTEP;
      if (r >= rows) break;
      const int grow = row_base + r;
      uint4 val = *reinterpret_cast<const uint4*>(stg + r * Cfg::OUT_PITCH + c * 16);
      bf16* dst = C + (long long)grow * ldc + col;
      if constexpr (ACT == ACT_ROPE) {
        const int gh = col >> 7, d = col & 127;
        const int which = gh / rp.H, head = gh - which * rp.H;
        if (which != 0) {
          int gb, col_c;   // cache clip and column of the row
          if (rp.pack != nullptr) {
            const int2 sp = __ldg(reinterpret_cast<const int2*>(pack_row(rp.pack, grow)));
            gb = __ldg(pack_slot(rp.pack) + sp.x); col_c = sp.y;
          } else {
            gb = grow / rp.S; col_c = rp.start_pos + grow - gb * rp.S;
          }
          dst = (which == 1 ? rp.kcache : rp.vcache) + d +
                (rp.pages.table != nullptr ? kv_paged_off(rp.pages, gb, head, col_c)   // paged: one more lookup
                                           : (((long long)gb * rp.H + head) * rp.s_max + col_c) * 128);
        }
      } else if (RES && residual != nullptr) {
        val.x = bf16x2_add(val.x, rr[u].x); val.y = bf16x2_add(val.y, rr[u].y);
        val.z = bf16x2_add(val.z, rr[u].z); val.w = bf16x2_add(val.w, rr[u].w);
      }
      *reinterpret_cast<uint4*>(dst) = val;
    }
  }
}

// CL = thread-block-cluster size along M (1, 2 or 4). The CL CTAs of a cluster work on CL
// consecutive M tiles of the SAME N tile: every CTA fetches 1/CL of the weight tile and TMA-multicasts
// it into all CL shared memories, so a weight byte crosses L2->SM once per cluster instead of once
// per CTA. A ring slot is refilled only once the consumers of EVERY CTA of the cluster have released it.
template <int BLOCK_N, int ACT, int CL>
__global__ void __launch_bounds__(384, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tmap_a,
                    const __grid_constant__ CUtensorMap tmap_b, bf16* C, long long ldc,
                    const bf16* __restrict__ bias, const bf16* residual, long long ldr, int M,
                    int N, int K, const RopeEpilogue rope) {
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int STAGES = Cfg::STAGES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;                 // 1024-byte aligned (SWIZZLE_128B atoms)
  const uint32_t smem_base = raw_addr + pad;

  // mbarriers (BAR_BYTES): full[STAGES] | empty[STAGES] | staged[2] | drained[2].
  //   full / empty : the operand ring; a consumer waits on full with the ring phase, the producer on empty with its
  //                  inverse.
  //   staged[cw]   : consumer warpgroup cw has written tile i's outputs to its staging block (128 arrivals); the
  //                  store warps wait with phase i & 1.
  //   drained[cw]  : the store warps have read that block out (96 arrivals); consumer warpgroup cw waits with
  //                  phase (i - 1) & 1 before it stages tile i > 0 into the same block.
  const uint32_t bar_base = smem_base + STAGES * Cfg::STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  auto staged_bar = [&](int cw) { return bar_base + 8u * (2 * STAGES + cw); };
  auto drained_bar = [&](int cw) { return bar_base + 8u * (2 * STAGES + 2 + cw); };
  uint8_t* stage_out = smem + STAGES * Cfg::STAGE_BYTES + Cfg::BAR_BYTES;

  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2 * CL);   // one arrival per consumer warpgroup of every CTA of the cluster
    }
    for (int cw = 0; cw < 2; ++cw) {
      mbar_init(staged_bar(cw), 128);
      mbar_init(drained_bar(cw), STORE_THREADS);
    }
    mbar_fence_init();
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();      // peers' barriers are initialised before anyone signals them

  const int num_m = (M + Cfg::BLOCK_M - 1) / Cfg::BLOCK_M;
  const int num_n = (N + BLOCK_N - 1) / BLOCK_N;
  const int num_k = (K + Cfg::BLOCK_K - 1) / Cfg::BLOCK_K;
  // cluster-tile = (N tile, group of CL M tiles); this CTA takes M tile `group*CL + rank`
  const int cta_rank = CL > 1 ? (int)cluster_ctarank() : 0;
  const int cluster_id = blockIdx.x / CL, n_clusters = gridDim.x / CL;
  const int num_tiles = ((num_m + CL - 1) / CL) * num_n;
  constexpr uint16_t MC_MASK = (uint16_t)((1u << CL) - 1u);
  constexpr int B_SLICE_ROWS = BLOCK_N / CL;

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<56>();    // the store warps keep RES_INFLIGHT residual chunks in registers
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = cluster_id; tile < num_tiles; tile += n_clusters) {
        const int m_blk = (tile / num_n) * CL + cta_rank, n_blk = tile % num_n;
        for (int kb = 0; kb < num_k; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);    // slot free in EVERY CTA of the cluster
          mbar_arrive_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
          const uint32_t a_dst = smem_base + stage * Cfg::STAGE_BYTES;
          tma_load_2d(a_dst, &tmap_a, full_bar(stage), kb * Cfg::BLOCK_K, m_blk * Cfg::BLOCK_M);
          if (CL == 1) {
            tma_load_2d(a_dst + Cfg::A_BYTES, &tmap_b, full_bar(stage), kb * Cfg::BLOCK_K, n_blk * BLOCK_N);
          } else {
            // my slice of the weight tile, delivered to the same offset in all CL shared memories
            tma_load_2d_mc(a_dst + Cfg::A_BYTES + cta_rank * B_SLICE_ROWS * 128, &tmap_b,
                           full_bar(stage), kb * Cfg::BLOCK_K, n_blk * BLOCK_N + cta_rank * B_SLICE_ROWS,
                           MC_MASK);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    } else if (threadIdx.x >= 32) {
      // ------------------------------ store warps ------------------------------
      const int t = threadIdx.x - 32;
      uint32_t phase = 0;
      for (int tile = cluster_id; tile < num_tiles; tile += n_clusters) {
        const int m_blk = (tile / num_n) * CL + cta_rank, n_blk = tile % num_n;
#pragma unroll 1
        for (int cw = 0; cw < 2; ++cw) {
          mbar_wait(staged_bar(cw), phase);
          gemm_epilogue_store<BLOCK_N, ACT>(stage_out + cw * 64 * Cfg::OUT_PITCH, t, m_blk * Cfg::BLOCK_M + cw * 64,
                                            n_blk, C, ldc, residual, ldr, M, N, rope);
          mbar_arrive(drained_bar(cw));
        }
        phase ^= 1u;
      }
    }
  } else {
    // ------------------------------ consumers: 64 rows each ------------------------------
    setmaxnreg_inc<224>();   // 56 * 128 + 224 * 256 = the 168 * 384 registers the CTA was launched with
    const int cw = wg - 1;
    const int t = threadIdx.x & 127, lane = threadIdx.x & 31, wq = t >> 5;
    uint8_t* stg = stage_out + cw * 64 * Cfg::OUT_PITCH;
    auto release = [&](int s) {
      if (t == 0) {
        if (CL == 1) {
          mbar_arrive(empty_bar(s));
        } else {
#pragma unroll
          for (int r = 0; r < CL; ++r) mbar_arrive_cluster(mapa_cluster(empty_bar(s), (uint32_t)r));
        }
      }
    };
    float acc[BLOCK_N / 2];
    int stage = 0;
    uint32_t phase = 0, out_phase = 0;
    for (int tile = cluster_id; tile < num_tiles; tile += n_clusters) {
      const int m_blk = (tile / num_n) * CL + cta_rank, n_blk = tile % num_n;
      int prev = -1;
      for (int kb = 0; kb < num_k; ++kb) {
        mbar_wait(full_bar(stage), phase);            // TMA bytes have landed
        const uint32_t a_addr = smem_base + stage * Cfg::STAGE_BYTES;
        const uint64_t a_desc = wgmma_desc_k_sw128(a_addr + cw * 64 * 128);
        const uint64_t b_desc = wgmma_desc_k_sw128(a_addr + Cfg::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < Cfg::BLOCK_K / 16; ++k) {
          // advance 16 bf16 = 32 B along K inside the swizzle span: +2 in the (addr >> 4) field
          wgmma_bf16<BLOCK_N>(acc, a_desc + 2u * k, b_desc + 2u * k, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                              // the previous k-block's wgmma has retired: its slot is free
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      release(prev);
      wgmma_fence_regs(acc);
      if (tile != cluster_id) {                       // the previous tile's staged block has been read out
        mbar_wait(drained_bar(cw), out_phase);
        out_phase ^= 1u;
      }
      gemm_epilogue_stage<BLOCK_N, ACT>(acc, stg, lane, wq, m_blk * Cfg::BLOCK_M + cw * 64, n_blk, bias, M, N, rope);
      mbar_arrive(staged_bar(cw));                    // hand the block to the store warps, start the next tile
    }
  }

  __syncthreads();                     // after the store warps' last store
  if (CL > 1) cluster_sync_all();      // nobody exits while a peer may still multicast / signal into it
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
static int resolve_encode() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
    set_last_error("cuTensorMapEncodeTiled is not available from the driver (%s)",
                   cudaGetErrorString(e));
    return -2;
  }
  g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  return 0;
}

// 2-D bf16 tensor [rows, cols] with row pitch ld (elements); box = [box_rows, 64 cols], 128B swizzle.
int make_tmap_2d(CUtensorMap* out, const void* ptr, long long rows, long long cols, long long ld,
                 int box_rows) {
  if (resolve_encode() != 0) return -2;
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim,
                        gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed (%d) ptr=%p rows=%lld cols=%lld ld=%lld box=%d",
                   (int)r, ptr, rows, cols, ld, box_rows);
    return -2;
  }
  return 0;
}

static int g_num_sms = 0;
int device_num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

template <int BLOCK_N, int ACT, int CL>
static int launch_one(const GemmArgs& g, cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N>;
  auto kern = gemm_bf16_tn_kernel<BLOCK_N, ACT, CL>;
  CUtensorMap ta, tb;
  if (make_tmap_2d(&ta, g.A, g.M, g.K, g.lda, Cfg::BLOCK_M) != 0) return -2;
  if (make_tmap_2d(&tb, g.W, g.N, g.K, g.ldw, BLOCK_N / CL) != 0) return -2;
  const int num_m = (g.M + 127) / 128;
  const int num_tiles = ((num_m + CL - 1) / CL) * ((g.N + BLOCK_N - 1) / BLOCK_N);   // cluster-tiles
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(384);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = CL > 1 ? 1 : 0;
  // persistent CTAs: as many clusters as are resident at once (GPC boundaries strand some SMs for clusters)
  static int resident = 0;
  if (resident == 0) {
    if (CL > 1) {
      cfg.gridDim = dim3(CL);
      VCL_CUDA_OK(cudaOccupancyMaxActiveClusters(&resident, kern, &cfg));
    }
    if (resident <= 0) resident = device_num_sms() / CL;
  }
  int clusters = resident;
  if (clusters > num_tiles) clusters = num_tiles;
  if (g.max_ctas > 0 && clusters * CL > g.max_ctas) clusters = g.max_ctas / CL > 0 ? g.max_ctas / CL : 1;
  cfg.gridDim = dim3(clusters * CL);
  VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, ta, tb, g.C, (long long)g.ldc, g.bias, g.residual,
                                 (long long)g.ldr, g.M, g.N, g.K, g.rope));
  count_launches(1);
  return 0;
}

template <int BLOCK_N, int ACT>
static int launch_cl(const GemmArgs& g, int cl, cudaStream_t stream) {
  if (BLOCK_N >= 128) {   // multicast slices must stay whole 8-row swizzle groups and >= 32 rows
    if (cl == 4) return launch_one<BLOCK_N, ACT, (BLOCK_N >= 128 ? 4 : 1)>(g, stream);
    if (cl == 2) return launch_one<BLOCK_N, ACT, (BLOCK_N >= 128 ? 2 : 1)>(g, stream);
  }
  return launch_one<BLOCK_N, ACT, 1>(g, stream);
}

template <int BLOCK_N>
static int launch_act(const GemmArgs& g, int cl, cudaStream_t stream) {
  switch (g.act) {
    case ACT_NONE: return launch_cl<BLOCK_N, ACT_NONE>(g, cl, stream);
    case ACT_QGELU: return launch_cl<BLOCK_N, ACT_QGELU>(g, cl, stream);
    case ACT_GELU: return launch_cl<BLOCK_N, ACT_GELU>(g, cl, stream);
    case ACT_SWIGLU: return launch_cl<BLOCK_N, ACT_SWIGLU>(g, cl, stream);
    case ACT_ROPE:
      if constexpr (BLOCK_N >= 128) return launch_cl<BLOCK_N, ACT_ROPE>(g, cl, stream);
      break;
  }
  set_last_error("gemm: unknown activation %d", g.act);
  return -1;
}

template <int BLOCK_N, int ACT>
static int init_one() {
  VCL_CUDA_OK(cudaFuncSetAttribute(gemm_bf16_tn_kernel<BLOCK_N, ACT, 1>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   GemmCfg<BLOCK_N>::SMEM_BYTES));
  if (BLOCK_N >= 128) {
    VCL_CUDA_OK(cudaFuncSetAttribute(gemm_bf16_tn_kernel<BLOCK_N, ACT, (BLOCK_N >= 128 ? 2 : 1)>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     GemmCfg<BLOCK_N>::SMEM_BYTES));
    VCL_CUDA_OK(cudaFuncSetAttribute(gemm_bf16_tn_kernel<BLOCK_N, ACT, (BLOCK_N >= 128 ? 4 : 1)>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     GemmCfg<BLOCK_N>::SMEM_BYTES));
  }
  return 0;
}
template <int BLOCK_N>
static int init_bn() {
  if (init_one<BLOCK_N, ACT_NONE>() || init_one<BLOCK_N, ACT_QGELU>() ||
      init_one<BLOCK_N, ACT_GELU>() || init_one<BLOCK_N, ACT_SWIGLU>()) return -2;
  if constexpr (BLOCK_N >= 128) {
    if (init_one<BLOCK_N, ACT_ROPE>()) return -2;
  }
  return 0;
}
int init_gemm_kernels() {
  if (resolve_encode() != 0) return -2;
  if (init_bn<256>() || init_bn<128>() || init_bn<64>() || init_bn<32>()) return -2;
  return 0;
}

int launch_gemm_bf16_tn(const GemmArgs& g, cudaStream_t stream) {
  VCL_REQUIRE(g.M > 0 && g.N > 0 && g.K > 0, "gemm: empty problem M=%d N=%d K=%d", g.M, g.N, g.K);
  VCL_REQUIRE(g.K % 64 == 0, "gemm: K=%d must be a multiple of 64", g.K);
  VCL_REQUIRE(g.N % 32 == 0, "gemm: N=%d must be a multiple of 32", g.N);
  VCL_REQUIRE(g.lda % 8 == 0 && g.ldw % 8 == 0 && g.ldc % 8 == 0, "gemm: pitches must be x8");
  const int n_out = g.act == ACT_SWIGLU ? g.N / 2 : g.N;
  VCL_REQUIRE(g.lda >= g.K && g.ldw >= g.K && g.ldc >= n_out && (g.residual == nullptr || g.ldr >= n_out),
              "gemm: pitches must cover a row (lda=%lld ldw=%lld >= K=%d, ldc=%lld ldr=%lld >= output width %d)",
              g.lda, g.ldw, g.K, g.ldc, g.ldr, n_out);
  VCL_REQUIRE(((uintptr_t)g.A % 16) == 0 && ((uintptr_t)g.W % 16) == 0 &&
                  ((uintptr_t)g.C % 16) == 0, "gemm: pointers must be 16-byte aligned");
  VCL_REQUIRE(g.residual == nullptr || (g.ldr % 8 == 0 && ((uintptr_t)g.residual % 16) == 0),
              "gemm: residual must be 16-byte aligned with pitch x8");
  VCL_REQUIRE(g.bias == nullptr || ((uintptr_t)g.bias % 16) == 0, "gemm: bias alignment");
  VCL_REQUIRE(!(g.act == ACT_SWIGLU && g.residual != nullptr), "gemm: swiglu takes no residual");
  if (g.act == ACT_ROPE) {
    const RopeEpilogue& r = g.rope;
    VCL_REQUIRE(r.cos_t && r.sin_t && r.kcache && r.vcache && r.S > 0 && r.H > 0, "gemm: ACT_ROPE needs the RoPE tables and the cache");
    VCL_REQUIRE(g.N == 3 * r.H * 128 && (r.pack != nullptr || g.M % r.S == 0) && r.start_pos + r.S <= r.s_max &&
                    g.bias == nullptr && g.residual == nullptr,
                "gemm: ACT_ROPE shape (N=%d, H=%d, M=%d, S=%d, start %d, cache %d)", g.N, r.H, g.M, r.S, r.start_pos, r.s_max);
    VCL_REQUIRE(((uintptr_t)r.kcache % 16) == 0 && ((uintptr_t)r.vcache % 16) == 0 && ((uintptr_t)r.cos_t % 16) == 0 &&
                    ((uintptr_t)r.sin_t % 16) == 0, "gemm: ACT_ROPE pointers must be 16-byte aligned");
  }
  int bn = g.block_n;
  int cl = g.cluster;
  if (bn == 0) {
    // Tile choice, from tools/sweep_gemm.py on an H100 80GB HBM3 at 400 W (DESIGN.md section 6). No cluster: the
    // multicast clusters (CL 2 / 4) were 1.5-3x slower than CL 1 at every shape the model runs.
    const int sms = device_num_sms();
    const long long mt = (g.M + 127) / 128;
    if (mt == 1) {
      // one M tile (decode beyond 16 clips): the narrowest tile that still gives every SM work
      bn = 256;
      while (bn > 32 && (g.N % bn != 0 || g.N / bn < sms)) bn >>= 1;
      if (g.N % bn != 0) bn = 32;
    } else if (g.N % 256 == 0 && mt * (g.N / 256) >= sms && !(g.N <= 1024 && g.K <= 1024)) {
      // enough 128 x 256 tiles for every SM: ViT qkv 305 vs 326 us (bn 128), fc1 463 vs 496, fc2 453 vs 461;
      // prefill M = 448 q|k|v 136 vs 139, gate|up 233 vs 292; M = 7168 o 463 vs 577, down 1173 vs 1656
      bn = 256;
    } else {
      // fewer 256-wide tiles than SMs (M = 448 o 46 vs 62 us, down 109 vs 140; projector 19 vs 27), or N = 1024 at
      // K <= 1024, where 4 N tiles of 256 leave a last wave 9 % full (ViT out 136 vs 146, patch-embed 65 vs 73)
      bn = (g.N % 128 == 0) ? 128 : (g.N % 64 == 0) ? 64 : 32;
    }
  }
  if (cl == 0) cl = 1;
  // cluster = -2: a CTA pair on one 256 x BLOCK_N tile, each CTA fetching half of the weight tile. sm_90 has no
  // pair MMA (each CTA's wgmma reads only its own shared memory), so the pair is the 2-CTA multicast cluster:
  // both halves land in both CTAs. Pairs take 128- or 256-wide tiles; anything else runs without a cluster.
  if (cl == -2) cl = (bn == 256 || bn == 128) && g.N % bn == 0 ? 2 : 1;
  if (g.act == ACT_ROPE && g.block_n == 0 && bn < 128) bn = 128;      // one head (128 columns) per tile at least
  VCL_REQUIRE(g.act != ACT_ROPE || bn == 128 || bn == 256, "gemm: ACT_ROPE needs 128- or 256-wide tiles (one head = 128 columns), got %d", bn);
  VCL_REQUIRE(cl == 1 || cl == 2 || cl == 4, "gemm: cluster must be 1, 2 or 4 (got %d)", cl);
  switch (bn) {
    case 256: return launch_act<256>(g, cl, stream);
    case 128: return launch_act<128>(g, cl, stream);
    case 64: return launch_act<64>(g, 1, stream);
    case 32: return launch_act<32>(g, 1, stream);
  }
  set_last_error("gemm: unsupported block_n %d", bn);
  return -1;
}

}  // namespace vcl

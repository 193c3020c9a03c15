// Attention kernels.
//
// (1) attn_fwd_kernel: softmax(Q K^T * scale [+causal]) V for full sequences (CLIP: S=257, hd=64,
//     non-causal; LLaMA prefill: S=S_p, hd=128, causal). Flash-style single pass, 64-query x
//     64-key tiles, cp.async double-buffered K/V in XOR-swizzled shared memory, bf16 mma.sync
//     (m16n8k16) with fp32 accumulation and fp32 online softmax.
//     Reference arithmetic: transformers/models/clip/modeling_clip.py:261-279 and
//     transformers/models/llama/modeling_llama.py:199-222 (eager): scores are a bf16 tensor that is
//     multiplied by `scaling` (a second bf16 rounding), softmax runs in fp32 and is cast back to
//     bf16 before the PV matmul. The score roundings are reproduced; the probabilities are rounded
//     to bf16 un-normalised (flash form), the one place this kernel differs from eager by design.
//     It serves the 336-px ViT tower (S = 577, read straight out of the fused q|k|v activation,
//     launch_attention_vit), longer prompts and continued prefills beyond 512 keys, and the chunks of prompts over
//     512 tokens in a paged cache (vcl_llm_slots_prefill_chunk: packed, each key tile read through the block
//     table, the same tiles and arithmetic as the one-shot prefill of the whole prompt) and text tails appended to
//     a paged slot past 512 keys (vcl_llm_slots_prefill_append: those of the contiguous continued prefill), and the
//     packed option continuations of candidate scoring past 512 keys on the contiguous cache
//     (vcl_llm_slots_score_append, the same tiles and masks again); the
//     ViT's S = 257 runs in
//     attention_tc.cu, the causal hd-128 prefill up to 512 keys in attention_prefill_tc.cu (both wgmma, exact
//     full-row softmax).
//
// (2) the single-query decode attention lives in decode_attention.cu (cluster of 4 CTAs per head).
#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                        uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                          uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                               uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int HD>
__device__ __forceinline__ uint32_t tile_addr(uint32_t base, int row, int chunk) {
  return base + row * (HD * 2) + (((chunk) ^ (row & 7)) << 4);
}

// Load a [64, HD] tile (rows row0.. of a [S, HD] strided matrix) into swizzled smem.
template <int HD>
__device__ __forceinline__ void load_tile(uint32_t sbase, const bf16* g, long long row_stride,
                                          int row0, int S) {
  constexpr int CH = HD / 8;
#pragma unroll
  for (int i = 0; i < (64 * CH) / 128; ++i) {
    const int idx = threadIdx.x + i * 128;
    const int r = idx / CH, c = idx % CH;
    const int gr = row0 + r;
    const bool ok = gr < S;
    const bf16* src = g + (long long)(ok ? gr : 0) * row_stride + c * 8;
    cp_async16(tile_addr<HD>(sbase, r, c), src, ok);
  }
}

// PAD (causal only): left-padded clips (a.n_pad): a real query (cache column >= n_pad[b]) attends keys n_pad[b] ..
// its own column, and a tile of real queries starts at the first key tile that holds a real key; a pad query
// attends causally
// PACK: packed sequences (a.pack, kernels.h): blockIdx.z is sequence i, whose pack_end_i - pack_start_i queries start
// at its row offset and sit at absolute positions start_i .. ; its keys are columns 0 .. end_i - 1 of slot_i (q_off =
// start_i, S_kv = end_i). Sequences with pack_len > 0 belong to the wgmma kernel and are skipped. On a paged cache
// (PAGED, a.pages) key tile jt is the 64 columns at offset (jt % 2) * 64 of block table[slot_i][jt / 2]; on the
// contiguous cache it is columns jt * 64 .. of clip slot_i (vcl_llm_slots_score_append: option continuations that
// end past 512 keys).
// A query tile covers the rows, walks the key tiles and applies the masks of the same tile of the contiguous kernel
// at the same q_off, S_kv: a continued prefill (vcl_llm_slots_prefill_append: a text tail at any start_i). For a
// chunk of a prompt (vcl_llm_slots_prefill_chunk), start_i is a multiple of 64, so these are also the tiles and
// masks of a one-shot prefill of the whole prompt (S = S_kv = end, q_off = 0): keys past end_i are past every query
// of the chunk too, so both mask them causally, and the zero-filled columns past end_i only meet P = 0.
template <int HD, bool CAUSAL, bool PAD = false, bool PACK = false, bool PAGED = false>
__global__ void __launch_bounds__(128) attn_fwd_kernel(const AttnArgs a) {
  static_assert((!PAGED || PACK) && (!PACK || (CAUSAL && !PAD && HD == 128)),
                "packed sequences: causal, unpadded hd-128 attention; a paged cache is read by packed sequences only");
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int TILE_BYTES = 64 * HD * 2;
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + TILE_BYTES;       // 2 buffers
  const uint32_t sV = sK + 2 * TILE_BYTES;   // 2 buffers

  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int S = a.S;                                        // queries
  int S_kv = a.S_kv > 0 ? a.S_kv : a.S;               // keys (a continued prefill attends to the cache too)
  int q_off = a.q_off;                                // absolute position of query 0 (causal mask)
  const int q0 = qt * 64;
  long long q_base = (long long)b * a.q_sb, o_base = (long long)b * a.o_sb;
  int slot = 0;
  if constexpr (PACK) {
    if (__ldg(pack_len(a.pack) + b) != 0) return;     // a wgmma sequence (before the first barrier: the CTA leaves)
    q_off = __ldg(pack_start(a.pack) + b);
    S_kv = __ldg(pack_end(a.pack) + b);
    S = S_kv - q_off;
    if (q0 >= S) return;
    const long long off = __ldg(pack_off(a.pack) + b);
    q_base = off * a.q_ss; o_base = off * a.o_ss;
    slot = __ldg(pack_slot(a.pack) + b);
  }
  const bf16* qg = a.q + q_base + (long long)h * a.q_sh;
  const bf16* kg = a.k + (PAGED ? 0 : (long long)(PACK ? slot : b) * a.k_sb) + (long long)h * a.k_sh;
  const bf16* vg = a.v + (PAGED ? 0 : (long long)(PACK ? slot : b) * a.v_sb) + (long long)h * a.v_sh;
  // key tile jt (keys jt * 64 ..; keys >= S_kv are zero-filled, never read)
  auto load_kv = [&](uint32_t sk, uint32_t sv, int jt) {
    if constexpr (PAGED) {
      const long long pg = (long long)__ldg(a.pages.table + slot * a.pages.row + (jt >> 1)) * a.pages.blk +
                           (long long)(jt & 1) * 64 * a.k_ss;
      load_tile<HD>(sk, kg + pg, a.k_ss, 0, S_kv - jt * 64);
      load_tile<HD>(sv, vg + pg, a.v_ss, 0, S_kv - jt * 64);
    } else {
      load_tile<HD>(sk, kg, a.k_ss, jt * 64, S_kv);
      load_tile<HD>(sv, vg, a.v_ss, jt * 64, S_kv);
    }
  };

  const int n_tiles_all = (S_kv + 63) / 64;
  const int n_tiles = CAUSAL ? min(n_tiles_all, (q_off + q0 + 63) / 64 + 1) : n_tiles_all;
  const int k_pad = PAD ? __ldg(a.n_pad + b) : 0;                    // first real key of the clip
  const int jt0 = (PAD && q_off + q0 >= k_pad) ? k_pad / 64 : 0;     // key tiles below hold pad keys only

  load_tile<HD>(sQ, qg, a.q_ss, q0, S);
  load_kv(sK, sV, jt0);
  cp_async_commit();

  uint32_t qf[HD / 16][4];
  float o[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.f, 0.f};
  const float scale = a.scale;
  const int qrow0 = q0 + warp * 16 + (lane >> 2);  // rows qrow0 and qrow0 + 8
  int kmin[2] = {0, 0};                             // key floor of the two rows
  if constexpr (PAD) {
    kmin[0] = qrow0 + q_off >= k_pad ? k_pad : 0;
    kmin[1] = qrow0 + 8 + q_off >= k_pad ? k_pad : 0;
  }

  for (int jt = jt0; jt < n_tiles; ++jt) {
    const int buf = (jt - jt0) & 1;
    if (jt + 1 < n_tiles) {
      load_kv(sK + (buf ^ 1) * TILE_BYTES, sV + (buf ^ 1) * TILE_BYTES, jt + 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();

    if (jt == jt0) {
#pragma unroll
      for (int kk = 0; kk < HD / 16; ++kk) {
        const int r = warp * 16 + (lane & 15);
        const int c = kk * 2 + (lane >> 4);
        ldsm_x4(tile_addr<HD>(sQ, r, c), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
      }
    }

    // ---- S = Q K^T (16 x 64 per warp) ----
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    const uint32_t kb = sK + buf * TILE_BYTES;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {  // pairs of 8-key blocks
        const int mi = lane >> 3;
        const int r = (jp * 2 + (mi >> 1)) * 8 + (lane & 7);
        const int c = kk * 2 + (mi & 1);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(tile_addr<HD>(kb, r, c), b0, b1, b2, b3);
        mma_bf16_16816(s[jp * 2], qf[kk], b0, b1);
        mma_bf16_16816(s[jp * 2 + 1], qf[kk], b2, b3);
      }
    }

    // ---- scale, mask, online softmax ----
    const int kbase = jt * 64 + 2 * (lane & 3);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int kidx = kbase + nb * 8 + (e & 1);
        const int qrow = qrow0 + (e >> 1) * 8;
        float x = bf16r(bf16r(s[nb][e]) * scale);
        if (kidx >= S_kv || (CAUSAL && kidx > qrow + q_off)) x = -INFINITY;
        if (PAD && kidx < kmin[e >> 1]) x = -INFINITY;
        s[nb][e] = x;
        mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
    }
    float corr[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      corr[r] = exp2f((m_run[r] - m_use[r]) * 1.4426950408889634f);
      m_run[r] = m_new;
      l_run[r] *= corr[r];
    }
    uint32_t pf[4][4];  // P as A fragments for 4 k-steps of 16 keys
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {
      float p[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        p[e] = exp2f((s[nb][e] - m_use[e >> 1]) * 1.4426950408889634f);
        ls[e >> 1] += p[e];
      }
      pf[nb >> 1][(nb & 1) * 2 + 0] = pack_bf16x2(p[0], p[1]);
      pf[nb >> 1][(nb & 1) * 2 + 1] = pack_bf16x2(p[2], p[3]);
    }
    l_run[0] += ls[0];
    l_run[1] += ls[1];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      o[i][0] *= corr[0]; o[i][1] *= corr[0];
      o[i][2] *= corr[1]; o[i][3] *= corr[1];
    }

    // ---- O += P V ----
    const uint32_t vb = sV + buf * TILE_BYTES;
#pragma unroll
    for (int t = 0; t < 4; ++t) {        // 16 keys per step
#pragma unroll
      for (int dp = 0; dp < HD / 16; ++dp) {  // pairs of 8-wide d blocks
        const int mi = lane >> 3;
        const int r = t * 16 + (mi & 1) * 8 + (lane & 7);
        const int c = dp * 2 + (mi >> 1);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(tile_addr<HD>(vb, r, c), b0, b1, b2, b3);
        mma_bf16_16816(o[dp * 2], pf[t], b0, b1);
        mma_bf16_16816(o[dp * 2 + 1], pf[t], b2, b3);
      }
    }
    __syncthreads();  // all warps done with this buffer before it is refilled
  }

  // ---- finalise: O / l, bf16, store ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  bf16* og = a.o + (PACK ? o_base : (long long)b * a.o_sb) + (long long)h * a.o_sh;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qrow = qrow0 + r * 8;
    if (qrow < S) {
      const float inv = 1.0f / l_run[r];
      bf16* dst = og + (long long)qrow * a.o_ss + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        *reinterpret_cast<uint32_t*>(dst + i * 8) =
            pack_bf16x2(o[i][r * 2] * inv, o[i][r * 2 + 1] * inv);
      }
    }
  }
}

template <int HD, bool CAUSAL, bool PAD = false, bool PACK = false, bool PAGED = false>
int launch_attn_t(const AttnArgs& a, cudaStream_t stream) {
  constexpr int SMEM = 5 * 64 * HD * 2;
  auto kern = attn_fwd_kernel<HD, CAUSAL, PAD, PACK, PAGED>;
  dim3 grid((a.S + 63) / 64, a.H, a.B);
  kern<<<grid, 128, SMEM, stream>>>(a);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace

int init_attention_kernels() {
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_fwd_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 64 * 64 * 2));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_fwd_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 64 * 64 * 2));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_fwd_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 64 * 128 * 2));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_fwd_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 64 * 128 * 2));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_fwd_kernel<128, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 64 * 128 * 2));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_fwd_kernel<128, true, false, true, true>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 64 * 128 * 2));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_fwd_kernel<128, true, false, true, false>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 64 * 128 * 2));
  if (init_attention_tc_kernels() != 0) return -2;
  return init_attention_prefill_tc_kernels();
}

int launch_attention(const AttnArgs& a, cudaStream_t stream) {
  VCL_REQUIRE(a.head_dim == 64 || a.head_dim == 128, "attention: head_dim %d unsupported", a.head_dim);
  VCL_REQUIRE(a.q_ss % 8 == 0 && a.k_ss % 8 == 0 && a.v_ss % 8 == 0 && a.q_sh % 8 == 0 &&
                  a.k_sh % 8 == 0 && a.v_sh % 8 == 0 && a.q_sb % 8 == 0 && a.k_sb % 8 == 0 &&
                  a.v_sb % 8 == 0 && a.o_ss % 2 == 0 && a.o_sh % 2 == 0 && a.o_sb % 2 == 0,
              "attention: strides must keep 16-byte row alignment");
  VCL_REQUIRE(a.n_pad == nullptr || (a.causal && a.head_dim == 128), "attention: left padding needs causal hd-128 attention");
  VCL_REQUIRE(a.pack == nullptr || (a.causal && a.head_dim == 128 && a.n_pad == nullptr && a.S <= 512),
              "attention: packed sequences need causal hd-128 attention over at most 512 keys, unpadded");
  VCL_REQUIRE(a.pack == nullptr || a.pack_tc || a.pack_flash, "attention: a packed launch runs at least one kernel");
  if (a.B <= 0 || a.H <= 0 || a.S <= 0) return 0;
  if (a.pack != nullptr) {   // wgmma: up to 512 keys; flash: chunks of longer prompts, tails past 512 keys
    if (a.pack_tc && launch_attention_prefill_tc(a, stream) != 0) return -1;
    if (!a.pack_flash) return 0;
    return a.pages.table != nullptr ? launch_attn_t<128, true, false, true, true>(a, stream)
                                    : launch_attn_t<128, true, false, true, false>(a, stream);
  }
  if (attention_prefill_tc_supported(a)) return launch_attention_prefill_tc(a, stream);   // LLaMA prefill up to 512 keys
  if (a.n_pad != nullptr) return launch_attn_t<128, true, true>(a, stream);
  if (a.head_dim == 64) {
    return a.causal ? launch_attn_t<64, true>(a, stream) : launch_attn_t<64, false>(a, stream);
  }
  return a.causal ? launch_attn_t<128, true>(a, stream) : launch_attn_t<128, false>(a, stream);
}

// qkv: [n_frames * S, 3*C] (q | k | v, heads of 64 contiguous), out: [n_frames * S, C]
int launch_attention_vit(const bf16* qkv, bf16* out, int n_frames, int S, int H, int C, cudaStream_t stream) {
  VCL_REQUIRE(C == H * 64, "attention_vit: head_dim must be 64");
  if (attention_vit_tc_supported(S)) return launch_attention_vit_tc(qkv, out, n_frames, S, H, C, stream);
  AttnArgs a;
  a.q = qkv;         a.q_sb = (long long)S * 3 * C; a.q_sh = 64; a.q_ss = 3 * C;
  a.k = qkv + C;     a.k_sb = a.q_sb; a.k_sh = 64; a.k_ss = 3 * C;
  a.v = qkv + 2 * C; a.v_sb = a.q_sb; a.v_sh = 64; a.v_ss = 3 * C;
  a.o = out;         a.o_sb = (long long)S * C; a.o_sh = 64; a.o_ss = C;
  a.B = n_frames; a.H = H; a.S = S; a.head_dim = 64; a.scale = 0.125f; a.causal = 0;
  return launch_attention(a, stream);
}

}  // namespace vcl

// Causal self-attention of the LLaMA prefill on the Hopper warpgroup tensor cores (head_dim 128, up to 512 keys).
//
// One CTA = one warpgroup per (clip, head, 64-query tile); causal: the tile needs the key blocks of 128 keys up to
// its last query only. Every operand is a K-major 128-byte-swizzled tile in shared memory (the layout TMA writes
// with CU_TENSOR_MAP_SWIZZLE_128B, built here by the threads themselves: [rows x 64 bf16] tiles, 16-byte chunk c of
// row r stored at chunk c ^ (r % 8)), so both products run on wgmma.mma_async from shared-memory descriptors:
//   S_j = Q . K_j^T   M64 x N128 x K128 (8 k-steps)      Q [64 x 128 d], K_j [128 keys x 128 d]
//   O  += P_j . V_j   M64 x N128 x K128 (8 k-steps)      P_j [64 x 128 keys], V_j^T [128 d x 128 keys]
// V is transposed on its way into shared memory, so no MN-major operand is needed.
//
// The softmax is the EXACT full-row softmax of the eager reference: pass 1 computes the scores of every key block
// for the row maximum, pass 2 computes them again, exponentiates against the final maximum, writes P as bf16 and
// accumulates O and the row sum. (The flash kernel of attention.cu rescales against a running maximum instead.)
//
// Arithmetic follows transformers/models/llama/modeling_llama.py:199-222 (eager): the scores are a bf16 tensor,
// multiplied by `scaling` into another bf16 tensor, masked, softmax in fp32, probabilities cast to bf16 for the
// P.V product. As in the other attention kernels of this library P is rounded before the normalisation.
#include "common.cuh"
#include "kernels.h"

#include <stdlib.h>

namespace vcl {

namespace {

constexpr int PA_THREADS = 128;                          // one warpgroup
constexpr int PA_MAX_KB = 4;                             // key blocks of 128: 512 keys
constexpr int PA_OFF_Q = 0;                              // Q: 2 tiles [64 x 64]      16 KB
constexpr int PA_OFF_K = PA_OFF_Q + 2 * 64 * 128;        // K: 2 tiles [128 x 64]     32 KB
constexpr int PA_OFF_VT = PA_OFF_K + 2 * 128 * 128;      // V^T: 2 tiles [128 x 64]   32 KB
constexpr int PA_OFF_P = PA_OFF_VT + 2 * 128 * 128;      // P: 2 tiles [64 x 64]      16 KB
constexpr int PA_SMEM = PA_OFF_P + 2 * 64 * 128 + 1024;  // + manual 1024-B alignment

__device__ __forceinline__ uint32_t pa_sw128(int row, int chunk) {   // byte offset inside a SW128 tile
  return (uint32_t)row * 128u + (uint32_t)((chunk ^ (row & 7)) << 4);
}

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// rows [row0, row0 + R) x 128 d of a strided matrix -> two swizzled [R x 64] tiles; rows >= n_rows are zero
template <int R>
__device__ __forceinline__ void pa_load_rows(uint8_t* dst, const bf16* g, long long ss, int row0, int n_rows) {
#pragma unroll 4
  for (int idx = threadIdx.x; idx < R * 16; idx += PA_THREADS) {
    const int r = idx >> 4, c = idx & 15;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (row0 + r < n_rows) v = *reinterpret_cast<const uint4*>(g + (long long)(row0 + r) * ss + c * 8);
    *reinterpret_cast<uint4*>(dst + (c >> 3) * (R * 128) + pa_sw128(r, c & 7)) = v;
  }
}

// V rows [key0, key0 + 128) -> V^T as two swizzled [128 d x 64 keys] tiles; keys >= n_keys are zero
__device__ __forceinline__ void pa_load_vt(uint8_t* dst, const bf16* g, long long ss, int key0, int n_keys) {
#pragma unroll 4
  for (int idx = threadIdx.x; idx < 128 * 16; idx += PA_THREADS) {
    const int key = idx & 127, c = idx >> 7;              // consecutive threads: consecutive keys, same 8 d
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (key0 + key < n_keys) v = *reinterpret_cast<const uint4*>(g + (long long)(key0 + key) * ss + c * 8);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint8_t* tile = dst + (key >> 6) * (128 * 128);
    const int kc = (key & 63) >> 3, ke = key & 7;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int d = c * 8 + e;
      const uint16_t h = (uint16_t)(e & 1 ? w[e >> 1] >> 16 : w[e >> 1] & 0xffffu);
      *reinterpret_cast<uint16_t*>(tile + pa_sw128(d, kc) + ke * 2) = h;
    }
  }
}

// acc = A[64 x 128] . B[128 x 128]^T over K = 128 (two swizzle spans of both operands)
__device__ __forceinline__ void pa_mma(float (&acc)[64], uint32_t a_base, int a_tile_bytes, uint32_t b_base,
                                       int b_tile_bytes, bool accumulate) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint64_t ad = wgmma_desc_k_sw128(a_base + (k >> 2) * a_tile_bytes) + 2u * (k & 3);
    const uint64_t bd = wgmma_desc_k_sw128(b_base + (k >> 2) * b_tile_bytes) + 2u * (k & 3);
    wgmma_bf16<128>(acc, ad, bd, (accumulate || k > 0) ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
}

// PAD: left-padded clips (a.n_pad): a real query (cache column >= n_pad[b]) attends keys n_pad[b] .. its own column,
// and a tile of real queries starts at the first key block that holds a real key; a pad query attends causally.
// PACK: packed sequences (a.pack): blockIdx.z is sequence i, whose S_i = pack_len_i queries start at its row offset,
// sit at absolute positions start_i .. end_i - 1 and attend keys 0 .. their own position of clip slot_i of the cache
// (S = S_i, q_off = start_i, S_kv = end_i): a whole prompt (start 0, end S_i) or a text tail appended to a cached
// sequence, each walking the tiles of the contiguous prefill at the same q_off; the grid covers the longest
// sequence, so a CTA whose query tile starts past S_i has nothing to do.
// PAGED (with PACK): a paged cache (a.pages). Key block kb of sequence i is the 128 columns of block
// table[slot_i][kb], rows 128 elements apart, so one key block of this kernel is exactly one page.
template <bool PAD, bool PACK, bool PAGED = false>
__global__ void __launch_bounds__(PA_THREADS)
attn_prefill_tc_kernel(const AttnArgs a, int S_kv) {
  static_assert(!PAGED || (PACK && !PAD), "a paged cache is read by packed prefills only");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;
  const uint32_t sbase = raw_addr + pad;

  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
  const int q0 = qt * 64;
  int S = a.S, q_off = a.q_off;
  long long q_base = (long long)b * a.q_sb, o_base = (long long)b * a.o_sb, kv_clip = b;
  if constexpr (PACK) {
    S = __ldg(pack_len(a.pack) + b);
    if (q0 >= S) return;                                 // before the first barrier: the whole CTA leaves
    const long long off = __ldg(pack_off(a.pack) + b);
    S_kv = __ldg(pack_end(a.pack) + b); q_off = __ldg(pack_start(a.pack) + b);
    q_base = off * a.q_ss; o_base = off * a.o_ss; kv_clip = __ldg(pack_slot(a.pack) + b);
  }
  const bf16* qg = a.q + q_base + (long long)h * a.q_sh;
  const bf16* kg = a.k + (PAGED ? 0 : kv_clip * a.k_sb) + (long long)h * a.k_sh;
  const bf16* vg = a.v + (PAGED ? 0 : kv_clip * a.v_sb) + (long long)h * a.v_sh;
  // key block kb: rows kb * 128 .. of the clip, or rows 0 .. of its page (paged; keys >= S_kv are zero either way)
  auto load_k = [&](int kb) {
    if constexpr (PAGED)
      pa_load_rows<128>(smem + PA_OFF_K, kg + (long long)__ldg(a.pages.table + kv_clip * a.pages.row + kb) * a.pages.blk,
                        a.k_ss, 0, S_kv - kb * 128);
    else
      pa_load_rows<128>(smem + PA_OFF_K, kg, a.k_ss, kb * 128, S_kv);
  };
  auto load_vt = [&](int kb) {
    if constexpr (PAGED)
      pa_load_vt(smem + PA_OFF_VT, vg + (long long)__ldg(a.pages.table + kv_clip * a.pages.row + kb) * a.pages.blk,
                 a.v_ss, 0, S_kv - kb * 128);
    else
      pa_load_vt(smem + PA_OFF_VT, vg, a.v_ss, kb * 128, S_kv);
  };
  // key blocks this tile touches: keys up to the absolute position of its last query
  const int last_key = min(S_kv - 1, q_off + min(q0 + 63, S - 1));
  const int n_kb = last_key / 128 + 1;
  const int k_pad = PAD ? __ldg(a.n_pad + b) : 0;                  // first real key of the clip
  const int kb0 = (PAD && q_off + q0 >= k_pad) ? k_pad / 128 : 0;     // key blocks below hold pad keys only

  pa_load_rows<64>(smem + PA_OFF_Q, qg, a.q_ss, q0, S);

  const int r0 = 16 * wq + (lane >> 2), c2 = 2 * (lane & 3);
  int qpos[2];                                           // absolute positions of this thread's two rows
  qpos[0] = q_off + q0 + r0;
  qpos[1] = qpos[0] + 8;
  int kmin[2] = {0, 0};                                  // key floor of the two rows
  if constexpr (PAD) {
    kmin[0] = qpos[0] >= k_pad ? k_pad : 0;
    kmin[1] = qpos[1] >= k_pad ? k_pad : 0;
  }
  const float scale = a.scale;
  float acc[64] = {};
  // scaled, rounded, masked score of accumulator element i of key block kb (reference rounding points)
  auto score = [&](int kb, int i) {
    const int key = kb * 128 + 8 * (i >> 2) + c2 + (i & 1);
    const float x = bf16r(bf16r(acc[i]) * scale);
    if (PAD && key < kmin[(i >> 1) & 1]) return -INFINITY;
    return (key >= S_kv || key > qpos[(i >> 1) & 1]) ? -INFINITY : x;
  };

  // ---- pass 1: row maxima over every key block ----
  float m[2] = {-INFINITY, -INFINITY};
  for (int kb = kb0; kb < n_kb; ++kb) {
    __syncthreads();                                     // previous readers of K are done
    load_k(kb);
    fence_async_smem();
    __syncthreads();
    pa_mma(acc, sbase + PA_OFF_Q, 64 * 128, sbase + PA_OFF_K, 128 * 128, false);
#pragma unroll
    for (int i = 0; i < 64; ++i) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], score(kb, i));
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
    m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
    if (m[r] == -INFINITY) m[r] = 0.f;                   // rows beyond S (all keys masked): P = 0
  }

  // ---- pass 2: P against the final maximum, O += P . V ----
  float o[64] = {};
  float l[2] = {0.f, 0.f};
  for (int kb = kb0; kb < n_kb; ++kb) {
    __syncthreads();                                     // previous readers of K / V^T / P are done
    load_k(kb);
    load_vt(kb);
    fence_async_smem();
    __syncthreads();
    pa_mma(acc, sbase + PA_OFF_Q, 64 * 128, sbase + PA_OFF_K, 128 * 128, false);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int i = 4 * j + 2 * hh;
        const float p0 = exp2f((score(kb, i) - m[hh]) * 1.4426950408889634f);
        const float p1 = exp2f((score(kb, i + 1) - m[hh]) * 1.4426950408889634f);
        l[hh] += p0 + p1;
        const int row = r0 + 8 * hh, col = 8 * j + c2;   // col = key inside the block
        *reinterpret_cast<uint32_t*>(smem + PA_OFF_P + (col >> 6) * (64 * 128) + pa_sw128(row, (col & 63) >> 3) +
                                     (col & 7) * 2) = pack_bf16x2(p0, p1);
      }
    }
    fence_async_smem();
    __syncthreads();
    pa_mma(o, sbase + PA_OFF_P, 64 * 128, sbase + PA_OFF_VT, 128 * 128, kb > kb0);
  }

  // ---- O / l -> bf16 ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  bf16* og = a.o + o_base + (long long)h * a.o_sh;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int qrow = q0 + r0 + 8 * hh;
    if (qrow < S) {
      const float inv = 1.0f / l[hh];
      bf16* dst = og + (long long)qrow * a.o_ss + c2;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
    }
  }
}

}  // namespace

int init_attention_prefill_tc_kernels() {
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_prefill_tc_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PA_SMEM));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_prefill_tc_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PA_SMEM));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_prefill_tc_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PA_SMEM));
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_prefill_tc_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   PA_SMEM));
  return 0;
}

// The shapes this kernel takes: causal, head_dim 128, at most 512 keys, 16-byte aligned rows.
bool attention_prefill_tc_supported(const AttnArgs& a) {
  const bool off = getenv("VCL_PREFILL_ATTN_FLASH") != nullptr;            // A/B: the mma.sync kernel (read per call, so
                                                                           // that a test can compare the two in one process)
  const int S_kv = a.S_kv > 0 ? a.S_kv : a.S;
  if (off || !a.causal || a.head_dim != 128 || S_kv > 128 * PA_MAX_KB || a.S <= 0) return false;
  if (a.q_off + a.S > S_kv) return false;                                 // every query sees its own key
  if (a.o_ss % 2 != 0 || a.o_sh % 2 != 0 || a.o_sb % 2 != 0 || ((uintptr_t)a.o % 4) != 0) return false;
  if (a.q_ss % 8 != 0 || a.q_sh % 8 != 0 || a.q_sb % 8 != 0 || a.k_ss % 8 != 0 || a.k_sh % 8 != 0 ||
      a.k_sb % 8 != 0 || a.v_ss % 8 != 0 || a.v_sh % 8 != 0 || a.v_sb % 8 != 0) return false;   // 16-byte row loads
  return ((uintptr_t)a.q % 16) == 0 && ((uintptr_t)a.k % 16) == 0 && ((uintptr_t)a.v % 16) == 0;
}

int launch_attention_prefill_tc(const AttnArgs& a, cudaStream_t stream) {
  const int S_kv = a.S_kv > 0 ? a.S_kv : a.S;
  dim3 grid((a.S + 63) / 64, a.H, a.B);
  VCL_REQUIRE(a.pages.table == nullptr || a.pack != nullptr, "prefill attention: a paged cache needs packed rows");
  if (a.pages.table != nullptr) attn_prefill_tc_kernel<false, true, true><<<grid, PA_THREADS, PA_SMEM, stream>>>(a, S_kv);
  else if (a.pack != nullptr) attn_prefill_tc_kernel<false, true><<<grid, PA_THREADS, PA_SMEM, stream>>>(a, S_kv);
  else if (a.n_pad != nullptr) attn_prefill_tc_kernel<true, false><<<grid, PA_THREADS, PA_SMEM, stream>>>(a, S_kv);
  else attn_prefill_tc_kernel<false, false><<<grid, PA_THREADS, PA_SMEM, stream>>>(a, S_kv);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

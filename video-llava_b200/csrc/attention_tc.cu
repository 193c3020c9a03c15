// Attention of the CLIP ViT on the Hopper warpgroup tensor cores (head_dim 64, non-causal, 129 <= S <= 257).
//
// One CTA per (frame, head), two warpgroups; warpgroup w takes the 64-query tiles w, w + 2, ... of the frame (three
// warpgroups fit in shared memory, but not in registers without spilling: measured slower).
// K (all keys of the head, up to 320 rows) and Q tiles arrive by TMA straight out of the fused q|k|v activation
// (2-D tensor map, 128-byte swizzle: one 64-wide head is exactly one swizzle span, so the tiles land in the K-major
// layout wgmma reads); V is transposed by the threads into K-major [64 d x 64 keys] tiles, keys >= S zero.
//   S = Q . K^T    wgmma M64 x N256 x K64 over keys [0, 256), plus M64 x N32 over keys [256, 288) when S > 256
//   O = P . V      wgmma M64 x N64, K = keys (16 k-steps, plus one for key 256), P from shared memory
// The whole score row of a query lives in registers, so the softmax is the EXACT full-row softmax of the eager
// reference (one pass, P against the final row maximum). Keys >= S (rows of the next frame, or TMA zero fill at the
// end of the tensor) are masked; queries >= S are computed and not stored.
//
// Arithmetic follows transformers/models/clip/modeling_clip.py:261-279 (eager): the scores are a bf16 tensor,
// multiplied by `scale` into another bf16 tensor, softmax in fp32, probabilities cast to bf16 for P.V. As in the
// other attention kernels of this library P is rounded before the normalisation.
#include "common.cuh"
#include "kernels.h"

#include <stdlib.h>

namespace vcl {

namespace {

constexpr int VA_WG = 2;                                 // warpgroups per CTA
constexpr int VA_THREADS = VA_WG * 128;
constexpr int VA_TILE = 64 * 128;                        // one [64 rows x 64 bf16] swizzled tile (8 KB)
constexpr int VA_KEY_TILES = 5;                          // keys [0, 320)
constexpr int VA_OFF_K = 0;                              // K: [320 keys x 64 d]
constexpr int VA_OFF_VT = VA_OFF_K + VA_KEY_TILES * VA_TILE;    // V^T: 5 tiles [64 d x 64 keys]
constexpr int VA_OFF_Q = VA_OFF_VT + VA_KEY_TILES * VA_TILE;    // Q: one tile per warpgroup
constexpr int VA_OFF_P = VA_OFF_Q + VA_WG * VA_TILE;            // P: 5 tiles [64 q x 64 keys] per warpgroup
constexpr int VA_OFF_BAR = VA_OFF_P + VA_WG * VA_KEY_TILES * VA_TILE;
constexpr int VA_SMEM = VA_OFF_BAR + 64 + 1024;          // + barriers + manual 1024-B alignment
static_assert(VA_SMEM <= 227 * 1024, "shared memory");

__device__ __forceinline__ uint32_t va_sw128(int row, int chunk) {
  return (uint32_t)row * 128u + (uint32_t)((chunk ^ (row & 7)) << 4);
}

__device__ __forceinline__ void named_bar_sync_wg(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

__global__ void __launch_bounds__(VA_THREADS, 1)
attn_vit_tc_kernel(const __grid_constant__ CUtensorMap tmap, const bf16* __restrict__ qkv, bf16* __restrict__ out,
                   int S, int H, int C) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;
  const uint32_t sbase = raw_addr + pad;
  const uint32_t kbar = sbase + VA_OFF_BAR;
  auto qbar = [&](int w) { return sbase + VA_OFF_BAR + 8u * (1 + w); };

  const int frame = blockIdx.x / H, h = blockIdx.x - frame * H;
  const int row0 = frame * S;                            // first row of this frame in the activation
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, lane = threadIdx.x & 31, wq = t >> 5;
  const int n_qt = (S + 63) / 64;
  const int n_kt = (S + 63) / 64;                        // K tiles that hold keys

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap);
    mbar_init(kbar, 1);
    for (int w = 0; w < VA_WG; ++w) mbar_init(qbar(w), 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(kbar, n_kt * VA_TILE);
    for (int i = 0; i < n_kt; ++i) tma_load_2d(sbase + VA_OFF_K + i * VA_TILE, &tmap, kbar, C + h * 64, row0 + 64 * i);
    for (int w = 0; w < VA_WG && w < n_qt; ++w) {
      mbar_arrive_expect_tx(qbar(w), VA_TILE);
      tma_load_2d(sbase + VA_OFF_Q + w * VA_TILE, &tmap, qbar(w), h * 64, row0 + 64 * w);
    }
  }
  // V^T: element (d, key) in tile key / 64, row d; keys >= S (and the unused rows of K's last tile) read as zero
  const bf16* vg = qkv + (long long)row0 * 3 * C + 2 * C + h * 64;
  for (int idx = threadIdx.x; idx < VA_KEY_TILES * 64 * 8; idx += VA_THREADS) {
    const int key = idx % (VA_KEY_TILES * 64), c = idx / (VA_KEY_TILES * 64);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (key < S) v = *reinterpret_cast<const uint4*>(vg + (long long)key * 3 * C + c * 8);
    const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
    uint8_t* tile = smem + VA_OFF_VT + (key >> 6) * VA_TILE;
    const int kc = (key & 63) >> 3, ke = key & 7;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const uint16_t hv = (uint16_t)(e & 1 ? w4[e >> 1] >> 16 : w4[e >> 1] & 0xffffu);
      *reinterpret_cast<uint16_t*>(tile + va_sw128(c * 8 + e, kc) + ke * 2) = hv;
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  mbar_wait(kbar, 0);

  const int r0 = 16 * wq + (lane >> 2), c2 = 2 * (lane & 3);
  const bool tail = S > 256;                             // keys [256, S): one more N32 block
  uint8_t* P = smem + VA_OFF_P + wg * VA_KEY_TILES * VA_TILE;
  const uint32_t p_addr = sbase + VA_OFF_P + wg * VA_KEY_TILES * VA_TILE;
  const uint32_t q_addr = sbase + VA_OFF_Q + wg * VA_TILE;
  uint32_t qphase = 0;
  float s[128], s2[16], o[32];
  for (int qt = wg; qt < n_qt; qt += VA_WG) {
    mbar_wait(qbar(wg), qphase);
    qphase ^= 1u;
    // ---- S = Q . K^T ----  (the accumulators are defined here, so they are not live across iterations)
#pragma unroll
    for (int i = 0; i < 128; ++i) s[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) s2[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t ad = wgmma_desc_k_sw128(q_addr) + 2u * k;
      wgmma_bf16<256>(s, ad, wgmma_desc_k_sw128(sbase + VA_OFF_K) + 2u * k, k > 0 ? 1u : 0u);
      if (tail) wgmma_bf16<32>(s2, ad, wgmma_desc_k_sw128(sbase + VA_OFF_K + 256 * 128) + 2u * k, k > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    wgmma_fence_regs(s2);
    named_bar_sync_wg(1 + wg);                           // every thread's wgmma has read Q and the previous P
    if (t == 0 && qt + VA_WG < n_qt) {                   // next query tile of this warpgroup
      mbar_arrive_expect_tx(qbar(wg), VA_TILE);
      tma_load_2d(q_addr, &tmap, qbar(wg), h * 64, row0 + 64 * (qt + VA_WG));
    }
    // ---- exact softmax over the full row ----  (the scaled scores are bf16 values: kept packed in pairs)
    auto sc = [&](float x, int key) { return key < S ? bf16r(bf16r(x) * 0.125f) : -INFINITY; };
    float m[2] = {-INFINITY, -INFINITY};
    uint32_t sp[64], sp2[8];
    auto pack_sc = [&](const float* a, int i, int key0) {     // pair i of a block whose first key is key0
      const int hh = i & 1, col = key0 + 8 * (i >> 1) + c2;
      const float x0 = sc(a[2 * i], col), x1 = sc(a[2 * i + 1], col + 1);
      m[hh] = fmaxf(m[hh], fmaxf(x0, x1));
      return pack_bf16x2(x0, x1);
    };
    if (tail) {
#pragma unroll
      for (int i = 0; i < 8; ++i) sp2[i] = pack_sc(s2, i, 256);
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) sp[i] = pack_sc(s, i, 0);
    float l[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
      m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
    }
    auto put_p = [&](uint32_t x2, int i, int key0) {        // P pair (row, col), (row, col + 1) as bf16
      const int hh = i & 1, row = r0 + 8 * hh, col = key0 + 8 * (i >> 1) + c2;
      const float p0 = exp2f((bf16lo(x2) - m[hh]) * 1.4426950408889634f);
      const float p1 = exp2f((bf16hi(x2) - m[hh]) * 1.4426950408889634f);
      l[hh] += p0 + p1;
      *reinterpret_cast<uint32_t*>(P + (col >> 6) * VA_TILE + va_sw128(row, (col & 63) >> 3) + (col & 7) * 2) =
          pack_bf16x2(p0, p1);
    };
#pragma unroll
    for (int i = 0; i < 64; ++i) put_p(sp[i], i, 0);
    if (tail) {
#pragma unroll
      for (int i = 0; i < 8; ++i) put_p(sp2[i], i, 256);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    named_bar_sync_wg(1 + wg);
    // ---- O = P . V ----
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk)
      wgmma_bf16<64>(o, wgmma_desc_k_sw128(p_addr + (kk >> 2) * VA_TILE) + 2u * (kk & 3),
                     wgmma_desc_k_sw128(sbase + VA_OFF_VT + (kk >> 2) * VA_TILE) + 2u * (kk & 3), kk > 0 ? 1u : 0u);
    if (tail)
      wgmma_bf16<64>(o, wgmma_desc_k_sw128(p_addr + 4 * VA_TILE), wgmma_desc_k_sw128(sbase + VA_OFF_VT + 4 * VA_TILE), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    // ---- O / l -> bf16 ----
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int q = qt * 64 + r0 + 8 * hh;
      if (q < S) {
        const float inv = 1.0f / l[hh];
        bf16* dst = out + (long long)(row0 + q) * C + h * 64 + c2;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(o[4 * j + 2 * hh] * inv, o[4 * j + 2 * hh + 1] * inv);
      }
    }
  }
}

}  // namespace

int init_attention_tc_kernels() {
  VCL_CUDA_OK(cudaFuncSetAttribute(attn_vit_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, VA_SMEM));
  return 0;
}

bool attention_vit_tc_supported(int S) {
  const bool off = getenv("VCL_VIT_ATTN_FLASH") != nullptr;   // A/B: the mma.sync kernel (read per call, so that
                                                              // a test can compare the two in one process)
  return !off && S >= 129 && S <= 257;
}

// qkv: [n_frames * S, 3*C] (q | k | v, heads of 64 contiguous), out: [n_frames * S, C]
int launch_attention_vit_tc(const bf16* qkv, bf16* out, int n_frames, int S, int H, int C, cudaStream_t stream) {
  VCL_REQUIRE(C == H * 64, "attention_vit_tc: head_dim must be 64");
  VCL_REQUIRE(S >= 129 && S <= 257, "attention_vit_tc: S=%d outside 129..257", S);
  VCL_REQUIRE(((uintptr_t)qkv % 16) == 0 && ((uintptr_t)out % 16) == 0, "attention_vit_tc: pointers must be 16-byte aligned");
  CUtensorMap tm;
  if (make_tmap_2d(&tm, qkv, (long long)n_frames * S, 3LL * C, 3LL * C, 64) != 0) return -2;
  attn_vit_tc_kernel<<<n_frames * H, VA_THREADS, VA_SMEM, stream>>>(tm, qkv, out, S, H, C);
  VCL_CUDA_OK(cudaGetLastError());
  count_launches(1);
  return 0;
}

}  // namespace vcl

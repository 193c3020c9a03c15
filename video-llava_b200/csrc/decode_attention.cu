// Single-query (decode) attention over the KV cache, split across a thread-block cluster.
//
// One query row per (clip, head) against kv_len cached keys: 2 * kv_len * 256 B of K/V per head
// (7.5 MB per layer for 32 heads at kv_len ~ 460) and almost no math -- HBM/L2-latency bound. A
// single CTA per head leaves 100 of 132 SMs idle and serialises three dependent phases, so each
// head is given a CLUSTER of 4 CTAs: every CTA owns a quarter of the keys, and the softmax
// statistics and the partial outputs are exchanged through distributed shared memory:
//
//   A  scores of my keys (16 lanes per key, 8 keys in flight per thread) -> local max
//      cluster barrier, global max = max over the 4 CTAs (ld.shared::cluster)
//   B  e = exp(s - max) for my keys -> local sum
//      cluster barrier, global sum
//   C  p = bf16(e / sum); partial out[128] += p * V over my keys
//      cluster barrier, rank 0 adds the 4 partial outputs in a fixed order and writes bf16
//
// The exchange preserves the reference's eager arithmetic exactly where it rounds
// (transformers/models/llama/modeling_llama.py:199-222): scores bf16(bf16(q.k) * scale), fp32
// softmax over ALL keys, probabilities rounded to bf16 after the normalisation, fp32 accumulate.
// Programmatic dependent launch lets the following o_proj GEMV prefetch its weights meanwhile.
#include "common.cuh"
#include "kernels.h"

namespace vcl {

namespace {

constexpr int DA_THREADS = 256;

// read a float at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ float ld_dsmem(const float* local, uint32_t rank) {
  uint32_t addr = smem_u32(local), remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(addr), "r"(rank));
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
  return v;
}

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* scratch) {
  v = is_max ? warp_max(v) : warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  float r = scratch[0];
#pragma unroll
  for (int w = 1; w < DA_THREADS / 32; ++w) r = is_max ? fmaxf(r, scratch[w]) : r + scratch[w];
  return r;
}

// DA_SPLIT = CTAs per (clip, head): 4 for few clips (latency: more CTAs than SMs are needed to fill the
// machine at all), 2 or 1 when clips x heads alone oversubscribe it (throughput: fewer barriers per byte).
// The keys of clip b, n_pad[b] .. kv_len + pos_dev[b] - 1 (kernels.h: decode positions), are split over the CTAs.
// PAGED: a paged cache (kernels.h: KvPages; clip b is cache slot b). The slot's table row is staged in shared
// memory, and key j of a CTA's range, at column lo + j, is read from row (lo + j) % 128 of block tbl[(lo + j) / 128].
template <int DA_SPLIT, bool PAGED = false>
__global__ void __launch_bounds__(DA_THREADS)
decode_attn_cluster_kernel(const bf16* __restrict__ q, long long q_ld, const bf16* __restrict__ kcache,
                           const bf16* __restrict__ vcache, bf16* __restrict__ o, long long o_ld, int H,
                           int s_max, int kv_len, int per_cap, float scale, const int* __restrict__ pos_dev,
                           int o_xwin, const int* __restrict__ n_pad, const KvPages pages) {
  extern __shared__ float sm[];
  float* sc = sm;                       // [per_cap] scores -> probabilities of my keys
  float* red = sm + per_cap;            // [16][128] partial outputs over the 16 key groups
  const int h = blockIdx.y, b = blockIdx.z;
  int* tbl = reinterpret_cast<int*>(red + 16 * 128 + 128 + 2 + 8);   // PAGED: [pages.row] the slot's table row
  if constexpr (PAGED) {
    // the table is constant while a decode graph runs (written before it, like pos_dev): read before the wait
    for (int i = threadIdx.x; i < pages.row; i += DA_THREADS) tbl[i] = __ldg(pages.table + b * pages.row + i);
  }
  // the clip's position and key floor live on the device (one captured graph for every position and padding);
  // they are constant while the graph runs, so they can be read before the dependency wait. The first k0
  // cache columns hold pad keys, which are neither read nor split
  if (pos_dev != nullptr) kv_len += __ldg(pos_dev + b);
  const int k0 = __ldg(n_pad + b);
  const int per = ((kv_len - k0 + DA_SPLIT - 1) / DA_SPLIT + 15) / 16 * 16;   // keys per CTA, multiple of 16
  float* outp = red + 16 * 128;         // [128] this CTA's partial output
  float* stat = outp + 128;             // [0] local max, [1] local sum
  float* scratch = stat + 2;            // [8]
  const uint32_t rank = cluster_ctarank();
  const int lo = k0 + (int)rank * per;
  const int n_loc = max(0, min(kv_len - lo, per));
  const long long coff = PAGED ? (long long)h * 128 * 128 : (((long long)b * H + h) * s_max + lo) * 128;
  const bf16* kc = kcache + coff;
  const bf16* vc = vcache + coff;
  // element offset of key j of my range (relative to kc / vc)
  auto key_off = [&](int j) -> long long {
    if constexpr (PAGED) {
      const int c = lo + j;
      return (long long)tbl[c >> 7] * pages.blk + (c & 127) * 128;
    } else {
      return (long long)j * 128;
    }
  };

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if constexpr (PAGED) __syncthreads();   // tbl is staged

  constexpr int U = 8;
  const int g = threadIdx.x >> 4, dc = threadIdx.x & 15;   // key slot (of 16) and 8-dim chunk
  // ---- A: scores ----
  {
    const uint4 qu = *reinterpret_cast<const uint4*>(q + (long long)b * q_ld + h * 128 + dc * 8);
    const float qf[8] = {bf16lo(qu.x), bf16hi(qu.x), bf16lo(qu.y), bf16hi(qu.y),
                         bf16lo(qu.z), bf16hi(qu.z), bf16lo(qu.w), bf16hi(qu.w)};
    // the trip count is the same for every lane (j0 - g, not j0): the two key slots of a warp would otherwise
    // part ways at the full-warp shuffles below when n_loc mod 128 is odd and < 16
    for (int j0 = g; j0 - g < n_loc; j0 += 16 * U) {
      uint4 ku[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int j = j0 + 16 * u;
        ku[u] = (j < n_loc) ? ld_nc_v4(kc + key_off(j) + dc * 8) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int j = j0 + 16 * u;
        float d = qf[0] * bf16lo(ku[u].x) + qf[1] * bf16hi(ku[u].x) + qf[2] * bf16lo(ku[u].y) +
                  qf[3] * bf16hi(ku[u].y) + qf[4] * bf16lo(ku[u].z) + qf[5] * bf16hi(ku[u].z) +
                  qf[6] * bf16lo(ku[u].w) + qf[7] * bf16hi(ku[u].w);
        d += __shfl_xor_sync(0xffffffffu, d, 8);
        d += __shfl_xor_sync(0xffffffffu, d, 4);
        d += __shfl_xor_sync(0xffffffffu, d, 2);
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        if (dc == 0 && j < n_loc) sc[j] = bf16r(bf16r(d) * scale);
      }
    }
  }
  // V loads of the first PV round do not depend on the softmax: issue them now
  uint4 vu[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int j = g + 16 * u;
    vu[u] = (j < n_loc) ? ld_nc_v4(vc + key_off(j) + dc * 8) : make_uint4(0, 0, 0, 0);
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < n_loc; j += DA_THREADS) mx = fmaxf(mx, sc[j]);
  mx = block_reduce(mx, true, scratch);
  if (threadIdx.x == 0) stat[0] = mx;
  cluster_sync_all();
  float gmax = -INFINITY;
#pragma unroll
  for (uint32_t r = 0; r < DA_SPLIT; ++r) gmax = fmaxf(gmax, ld_dsmem(&stat[0], r));
  // ---- B: exponentials and the global sum ----
  float sum = 0.f;
  for (int j = threadIdx.x; j < n_loc; j += DA_THREADS) {
    const float e = __expf(sc[j] - gmax);
    sc[j] = e;
    sum += e;
  }
  sum = block_reduce(sum, false, scratch);
  if (threadIdx.x == 0) stat[1] = sum;
  cluster_sync_all();
  float gsum = 0.f;
#pragma unroll
  for (uint32_t r = 0; r < DA_SPLIT; ++r) gsum += ld_dsmem(&stat[1], r);
  const float inv = 1.0f / gsum;
  // ---- C: partial output over my keys ----
  {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j0 = g; j0 < n_loc; j0 += 16 * U) {
      if (j0 != g) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int j = j0 + 16 * u;
          vu[u] = (j < n_loc) ? ld_nc_v4(vc + key_off(j) + dc * 8) : make_uint4(0, 0, 0, 0);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int j = j0 + 16 * u;
        const float p = (j < n_loc) ? bf16r(sc[j] * inv) : 0.f;
        acc[0] += p * bf16lo(vu[u].x); acc[1] += p * bf16hi(vu[u].x);
        acc[2] += p * bf16lo(vu[u].y); acc[3] += p * bf16hi(vu[u].y);
        acc[4] += p * bf16lo(vu[u].z); acc[5] += p * bf16hi(vu[u].z);
        acc[6] += p * bf16lo(vu[u].w); acc[7] += p * bf16hi(vu[u].w);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) red[g * 128 + dc * 8 + e] = acc[e];
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) v += red[k * 128 + threadIdx.x];
    outp[threadIdx.x] = v;
  }
  cluster_sync_all();
  if (rank == 0 && threadIdx.x < 128) {
    float v = 0.f;
#pragma unroll
    for (uint32_t r = 0; r < DA_SPLIT; ++r) v += ld_dsmem(&outp[threadIdx.x], r);
    const int col = h * 128 + threadIdx.x;
    const long long oo = o_xwin ? (long long)xwin_offset(b, col, (int)gridDim.z) : (long long)b * o_ld + col;
    o[oo] = __float2bfloat16_rn(v);
  }
  cluster_sync_all();   // keep every CTA's shared memory alive until rank 0 has read it
}

// CTAs per (clip, head): enough CTAs to cover the SMs a few times over, no more
int decode_split(int B, int H) {
  const long long heads = (long long)B * H;
  return heads <= 2 * device_num_sms() ? 4 : (heads <= 3 * device_num_sms() ? 2 : 1);
}

// dynamic shared memory of a launch whose CTAs hold the scores of up to kv_cap keys between them: the scores of a
// CTA's share, the 16 x 128 partial outputs, its partial output, the statistics, the reduction scratch and, paged,
// the slot's table row
size_t decode_smem(int split, int kv_cap, int table_row) {
  const int per = ((kv_cap + split - 1) / split + 15) / 16 * 16;   // keys per CTA, multiple of 16
  return (size_t)(per + 16 * 128 + 128 + 2 + 8 + table_row) * sizeof(float);
}

constexpr size_t DA_SMEM_MAX = 48 * 1024;

}  // namespace

bool decode_attention_fits(int B, int H, int s_max, bool paged) {
  return decode_smem(decode_split(B, H), s_max, paged ? (s_max + 127) / 128 : 0) <= DA_SMEM_MAX;
}

int launch_decode_attention(const bf16* q, long long q_ld, const bf16* kcache, const bf16* vcache,
                            bf16* o, long long o_ld, int B, int H, int head_dim, int s_max,
                            int kv_len, float scale, cudaStream_t stream, const int* pos_dev, bool o_xwin,
                            const int* n_pad, const KvPages& pages) {
  VCL_REQUIRE(head_dim == 128, "decode attention: head_dim must be 128");
  const bool paged = pages.table != nullptr;
  VCL_REQUIRE(!paged || pages.row == (s_max + 127) / 128, "decode attention: table rows of %d blocks for max_seq %d",
              pages.row, s_max);
  VCL_REQUIRE(n_pad != nullptr, "decode attention: needs the key floors n_pad");
  VCL_REQUIRE(kv_len > 0 && kv_len <= s_max, "decode attention: kv_len %d out of range", kv_len);
  // shared memory is sized for the longest sequence when the length is only known on the device
  const int kv_cap = pos_dev != nullptr ? s_max : kv_len;
  const int split = decode_split(B, H);
  const int per = ((kv_cap + split - 1) / split + 15) / 16 * 16;   // keys per CTA, multiple of 16
  const size_t smem = decode_smem(split, kv_cap, paged ? pages.row : 0);
  VCL_REQUIRE(smem <= DA_SMEM_MAX, "decode attention: %s %d too long for the smem budget (%zu of %zu bytes at %d "
              "CTAs per head for %d clips x %d heads%s)", pos_dev != nullptr ? "s_max" : "kv_len", kv_cap, smem,
              DA_SMEM_MAX, split, B, H, paged ? ", paged" : "");
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(split, H, B);
  cfg.blockDim = dim3(DA_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = split;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  auto kern = paged ? decode_attn_cluster_kernel<4, true> : decode_attn_cluster_kernel<4>;
  if (split == 2) kern = paged ? decode_attn_cluster_kernel<2, true> : decode_attn_cluster_kernel<2>;
  if (split == 1) kern = paged ? decode_attn_cluster_kernel<1, true> : decode_attn_cluster_kernel<1>;
  VCL_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, q, q_ld, kcache, vcache, o, o_ld, H, s_max, kv_len, per, scale, pos_dev,
                                 o_xwin ? 1 : 0, n_pad, pages));
  count_launches(1);
  return 0;
}

}  // namespace vcl

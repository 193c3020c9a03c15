// Internal launcher prototypes shared between the kernel translation units and vcl_api.cu.
// Everything here enqueues on the stream it is given and never synchronises.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vcl {

typedef __nv_bfloat16 bf16;

// Packed prefill (vcl_llm_slots_prefill / _chunk / _append): n <= PACK_SEQ_MAX sequences of lengths
// S_0 .. S_{n-1} concatenated without padding into M = sum S_i rows, sequence i going to cache slot slot_i. Sequence
// i is the rows start_i .. start_i + S_i - 1 of its prompt (start_i = 0 for a whole prompt; a chunk of a longer
// prompt, or a text tail appended to a kept conversation, attends the columns 0 .. start_i - 1 already in the
// cache). One device int array describes
// the layout, and every kernel of a packed prefill reads it through the accessors below:
//   [0, 64)    row offset of sequence i     [64, 128)   S_i when the wgmma prefill attention attends it, 0 when the
//                                                       flash kernel does (a chunk of a prompt over 512 tokens,
//                                                       or an appended tail that ends past 512 keys)
//   [128, 192) its cache slot               [192, 256)  its last row (offset + S_i - 1), whose logits give its token
//   [256, 320) start_i                      [320, 384)  start_i + S_i: the position of the token its last row gives
//   [384 + 2r] sequence of row r            [384 + 2r + 1] position of row r in its prompt (start_i + row in sequence)
constexpr int PACK_SEQ_MAX = 64;
constexpr int PACK_HEAD = 6 * PACK_SEQ_MAX;
inline size_t pack_elems(long long rows) { return PACK_HEAD + 2 * (size_t)rows; }
template <class T> __host__ __device__ inline T* pack_off(T* p) { return p; }
template <class T> __host__ __device__ inline T* pack_len(T* p) { return p + PACK_SEQ_MAX; }
template <class T> __host__ __device__ inline T* pack_slot(T* p) { return p + 2 * PACK_SEQ_MAX; }
template <class T> __host__ __device__ inline T* pack_last(T* p) { return p + 3 * PACK_SEQ_MAX; }
template <class T> __host__ __device__ inline T* pack_start(T* p) { return p + 4 * PACK_SEQ_MAX; }
template <class T> __host__ __device__ inline T* pack_end(T* p) { return p + 5 * PACK_SEQ_MAX; }
template <class T> __host__ __device__ inline T* pack_row(T* p, long long r) { return p + PACK_HEAD + 2 * r; }   // [seq, pos]

// Paged KV cache (vcl_config.kv_blocks > 0): one pool of blocks instead of the contiguous [clip][head][s_max][128]
// cache of a layer. A block is 128 columns of one sequence across all layers, [layer][K = 0 | V = 1][head][128][128]
// bf16 (blk elements). Column c of cache slot s lives in block table[s * row + c / 128] at offset c % 128, so with
// the K (or V) base of a layer, pool + (2 * layer (+ 1)) * H * 128 * 128, element (s, head, c, d) is at
// base + kv_paged_off(p, s, head, c) + d. A null table is the contiguous cache.
struct KvPages {
  const int* table = nullptr;   // [slots][row] block indices
  int row = 0;                  // ceil(s_max / 128)
  long long blk = 0;            // elements per block
};
__device__ __forceinline__ long long kv_paged_off(const KvPages& p, int slot, int head, int col) {
  return (long long)__ldg(p.table + slot * p.row + (col >> 7)) * p.blk + ((long long)head * 128 + (col & 127)) * 128;
}

enum Act { ACT_NONE = 0, ACT_QGELU = 1, ACT_GELU = 2, ACT_SWIGLU = 3, ACT_ROPE = 4 };
// ACT_ROPE: the GEMM is the LLaMA q|k|v projection of a prefill (N = 3 * H * 128, rows = [clip][position], or the
// packed rows of `pack`). The epilogue rotates q and k (RoPE, every product and the sum rounded to bf16 like the
// reference), writes q to C (columns [0, H * 128)), k and v straight into the KV cache; the k | v columns of C are
// not written.
struct RopeEpilogue {
  const bf16* cos_t = nullptr; const bf16* sin_t = nullptr;    // [s_max][64]
  bf16* kcache = nullptr; bf16* vcache = nullptr;              // [clip][head][s_max][128] of this layer
  int S = 0, start_pos = 0, H = 0, s_max = 0;                  // rows per clip, position of row 0, heads
  const int* n_pad = nullptr;                                  // [clip] left padding (see below) or null
  const int* pack = nullptr;   // packed rows (above) or null: row r is rotated by its position p and lands at
                               // column p of its sequence's slot (S, start_pos and n_pad are then unused)
  KvPages pages;               // packed rows only: a paged cache (kcache / vcache are then the layer's pool bases)
};

// Positions in the KV cache. Left padding (a batch of prompts of different lengths): clip b's first n_pad[b]
// cache columns hold pad tokens, column c holds RoPE position max(c - n_pad[b], 0), a query at column
// c >= n_pad[b] attends keys n_pad[b] .. c, and a pad query attends causally from key 0 (its output is unused but
// finite). Every `n_pad` below is a device array [clip]; the prefill kernels take null for no padding, the decode
// kernels always take one (all zeros for an unpadded cache). A decode token of clip b goes to column
// c_b = pos + (pos_dev ? pos_dev[b] : 0) (pos a host int, pos_dev a device array [clip]): it is rotated by the
// angle of max(c_b - n_pad[b], 0), appended at column c_b and attends keys n_pad[b] .. c_b. Both arrays are read
// on the device, so one captured decode graph serves every prompt length, padding and set of per-clip positions.

void set_last_error(const char* fmt, ...);
void count_launches(long long n);
long long launch_count();
int device_num_sms();

// ---- gemm_tc.cu : C[M,N] = epi(A[M,K] . W[N,K]^T), wgmma + TMA ----------------------------------
struct GemmArgs {
  const bf16* A = nullptr;  long long lda = 0;   // activations, row pitch in elements
  const bf16* W = nullptr;  long long ldw = 0;   // weights [N,K] (nn.Linear layout)
  bf16* C = nullptr;        long long ldc = 0;   // output (width N, or N/2 for ACT_SWIGLU)
  const bf16* bias = nullptr;                    // [N] or null
  const bf16* residual = nullptr; long long ldr = 0;  // [M,N] or null; may alias C
  int M = 0, N = 0, K = 0;
  int act = ACT_NONE;
  int block_n = 0;     // 0 = choose
  int cluster = 0;     // CTAs per cluster along M sharing multicast weight tiles: 0/1, 2 or 4
  int max_ctas = 0;    // 0 = one per SM
  RopeEpilogue rope;   // act == ACT_ROPE only
};
int launch_gemm_bf16_tn(const GemmArgs& g, cudaStream_t stream);
int init_gemm_kernels();
// 2-D bf16 tensor map [rows, cols] with row pitch ld (elements); box = [box_rows, 64], 128-B swizzle
int make_tmap_2d(CUtensorMap* out, const void* ptr, long long rows, long long cols, long long ld,
                 int box_rows);

// ---- elementwise.cu ---------------------------------------------------------------------------
// y = LayerNorm(x) * w + b   (rows x D, fp32 statistics, one bf16 rounding)
int launch_layernorm(const bf16* x, long long ldx, bf16* y, long long ldy, const bf16* w,
                     const bf16* b, int rows, int D, float eps, cudaStream_t stream);
// y = w * bf16(x * rsqrt(mean(x^2)+eps))   (LlamaRMSNorm rounding order)
int launch_rmsnorm(const bf16* x, long long ldx, bf16* y, long long ldy, const bf16* w, int rows,
                   int D, float eps, cudaStream_t stream);
// pixels -> patch matrix [N*P, KP] (k = c*ps*ps + i*ps + j, zero padded to KP)
//   mode 0: bf16 NCHW already normalised;  mode 1: uint8 NHWC raw, CLIP mean/std applied here
int launch_im2col(const void* pixels, int mode, bf16* out, int n_frames, int image, int patch,
                  int KP, cudaStream_t stream);
// h[n, 0] = LN(cls + pos[0]); h[n, 1+p] = LN(patch[n*P+p] + pos[1+p])
int launch_clip_embed_ln(const bf16* patch_out, const bf16* cls, const bf16* pos, const bf16* ln_w,
                         const bf16* ln_b, bf16* h, int n_frames, int P, int D, float eps,
                         cudaStream_t stream);
// token-embedding gather with the projected video rows spliced in after <vid_start>. pack (packed rows, M = B * S
// when null): row r is position p of sequence i, takes vid_start[i] and video row block i
int launch_embed_splice(const long long* ids, const bf16* table, const bf16* vid, const int* vid_start,
                        bf16* h, int B, int S, int D, int n_vid, int vocab, cudaStream_t stream,
                        const int* pack = nullptr, int M = 0);
// cos/sin tables [max_pos, head_dim/2] rounded to bf16 (stored as bf16)
int launch_rope_table(bf16* cos_t, bf16* sin_t, int max_pos, int head_dim, float theta,
                      cudaStream_t stream);
// prefill: rotate q (in place inside qkv) and k, write k/v into the cache at [pos0, pos0+S) (decode beyond 16
// clips: S = 1 at the decode positions above)
int launch_rope_kv_prefill(bf16* qkv, bf16* kcache, bf16* vcache, const bf16* cos_t,
                           const bf16* sin_t, int B, int S, int H, int head_dim, int s_max, int pos0,
                           cudaStream_t stream, const int* pos_dev = nullptr, const int* n_pad = nullptr);
// h[b,:] = table[tok[b*tok_stride]]  (decode-time embedding lookup, tokens live on the device)
int launch_embed_tokens(const int* tok, long long tok_stride, const bf16* table, bf16* h, int B,
                        int D, int vocab, cudaStream_t stream);
int launch_argmax(const float* logits, int* out, long long out_stride, int B, int V,
                  cudaStream_t stream);
int launch_fill_int(int* dst, int value, int n, cudaStream_t stream);   // dst[0 .. n) = value

// ---- st_pool.cu ---------------------------------------------------------------------------------
// dtype codes: 0 = fp16, 1 = bf16
int launch_st_pool(const void* feats, int in_dtype, long long frame_stride, long long patch_stride,
                   int T, int P, int C, int n_temporal, void* out, int out_dtype,
                   cudaStream_t stream);

// ---- cross_entropy.cu ---------------------------------------------------------------------------
// Rows row0 .. row0+rows-1 of a labelled batch whose logits [rows, ld] (first V columns) are at `logits`:
// nll[i] = -bf16(log_softmax(row i)[label]) (0 for label -100 or no target, NaN for a label outside 0..V-1),
// and logits_out [rows, V] (optional) the compact copy. Labels: labels[row] (seg == 0), or HF's shift over
// clips of seg columns: row = clip * seg + column, scored against labels[row + 1]; the last column of a clip
// has no target. nll may be null (labels may then be null too).
int launch_cross_entropy(const bf16* logits, long long ld, int V, const long long* labels, long long row0, int rows,
                         int seg, float* nll, bf16* logits_out, cudaStream_t stream);
// loss_out[0] = mean of nll[0 .. rows) over the rows with a target (NaN when there is none), fixed order;
// nll_out (optional): a copy of nll, [rows] (seg == 0) or [clip][seg - 1] (the last column of each clip dropped)
int launch_nll_mean(const float* nll, const long long* labels, long long rows, int seg, float* nll_out,
                    float* loss_out, cudaStream_t stream);

// ---- sampling.cu --------------------------------------------------------------------------------
// Next token of each logits row [B][ld] (first V columns; bf16 values in fp32 storage) by the rules at the top of
// sampling.cu. Row r uses entry t = entry0 + (rowmap ? rowmap[r] : r) of the sampling table (temperature, top_k,
// seed: device arrays; temperature 0 is greedy) and draws at counter p = col + (col_dev ? col_dev[r] : 0) -
// (n_pad ? n_pad[t] : 0), the RoPE position its token takes. out[r * out_stride] receives the token.
// Log-probs: an entry with top_n[t] >= 0 (top_n null: none) also writes places 0 .. top_n[t] of its row (place 0 the
// chosen token, then the alternatives), place q of the token at position p (0 <= p < lp_rows) at index
// t * lp_entry + p * lp_pos + q of lp_id / lp_val.
#ifndef VCL_LOGPROBS_MAX
#define VCL_LOGPROBS_MAX 20   // include/vcl.h
#endif
// The 32-bit path (top_p set; V <= VCL_SAMPLE_WIDE_MAX_V): entry t also has top_p[t] (1: off) and the repetition
// penalty rep[t] (1: off), applied to the tokens of its set, bitmap tset[t * tset_words ..] (null: every set empty),
// to which the sampler adds the token it picks.
#ifndef VCL_SAMPLE_WIDE_MAX_V
#define VCL_SAMPLE_WIDE_MAX_V 57344   // include/vcl.h
#endif
struct SampleArgs {
  const float* logits = nullptr; long long ld = 0; int V = 0, B = 0;
  const float* temperature = nullptr; const int* top_k = nullptr; const unsigned long long* seed = nullptr;
  int entry0 = 0; const int* rowmap = nullptr;
  int col = 0; const int* col_dev = nullptr; const int* n_pad = nullptr;
  int* out = nullptr; long long out_stride = 1;
  const int* top_n = nullptr;
  int* lp_id = nullptr; float* lp_val = nullptr;
  long long lp_entry = 0, lp_pos = 0; int lp_rows = 0;
  const float* top_p = nullptr; const float* rep = nullptr;
  unsigned int* tset = nullptr; int tset_words = 0;
};
int launch_sample(const SampleArgs& a, cudaStream_t stream);
// one token set: dst[0 .. words) cleared, then the bits of ids[0 .. n) (device int64; ids outside 0 .. V-1 ignored)
// set, in one launch
int launch_token_set(unsigned int* dst, int words, const long long* ids, int n, int V, cudaStream_t stream);

// ---- attention.cu -------------------------------------------------------------------------------
// softmax(Q K^T * scale [+ causal]) V for S_q == S_kv, bf16, fp32 softmax; element (b,h,s,d) of
// each operand lives at base + b*sb + h*sh + s*ss + d.
struct AttnArgs {
  const bf16* q; long long q_sb, q_sh, q_ss;
  const bf16* k; long long k_sb, k_sh, k_ss;
  const bf16* v; long long v_sb, v_sh, v_ss;
  bf16* o;       long long o_sb, o_sh, o_ss;
  int B, H, S, head_dim;
  float scale;
  int causal;
  int S_kv = 0;      // number of keys (0: = S); > S when the queries continue a cached sequence
  int q_off = 0;     // absolute position of query 0 for the causal mask (S_kv - S for a continuation)
  const int* n_pad = nullptr;   // causal only: [B] left padding, the key floor of real queries (or null)
  // packed rows (kernels.h, above) or null. Sequence i (i < B) has S = S_i, q_off = start_i, S_kv = start_i + S_i:
  // its queries / outputs are rows offset_i .. of q / o (q_sb, o_sb unused), its keys / values clip slot_i of k / v.
  // a.S is max S_i.
  // The wgmma kernel (S_i <= 512) whatever VCL_PREFILL_ATTN_FLASH says, for every sequence with pack_len S_i > 0.
  const int* pack = nullptr;
  // packed rows only: a paged cache. Key block kb of sequence i is block table[slot_i][kb] (k / v: the layer's pool
  // bases, k_sh / v_sh the head stride inside a block, k_ss = v_ss = 128; k_sb / v_sb unused)
  KvPages pages;
  // packed rows on a paged cache: which kernels run. pack_tc: the wgmma kernel for the sequences with pack_len > 0;
  // pack_flash: the flash kernel (attention.cu) for those with pack_len 0, whose queries start_i .. end_i - 1 attend
  // keys 0 .. their own position (one launch per kernel, each over every sequence; the other kind's CTAs leave)
  bool pack_tc = true, pack_flash = false;
};
int launch_attention(const AttnArgs& a, cudaStream_t stream);     // dispatches to the wgmma prefill kernel when it applies
int init_attention_kernels();
// ---- attention_prefill_tc.cu : wgmma causal attention (hd 128, <= 512 keys, exact full-row softmax) ----
bool attention_prefill_tc_supported(const AttnArgs& a);
int launch_attention_prefill_tc(const AttnArgs& a, cudaStream_t stream);
int init_attention_prefill_tc_kernels();
// the ViT's attention (hd 64, non-causal) straight out of the fused q|k|v activation [n_frames * S, 3*C]:
// the wgmma kernel below for 129 <= S <= 257, the mma.sync kernel otherwise (336-px tower, S = 577)
int launch_attention_vit(const bf16* qkv, bf16* out, int n_frames, int S, int H, int C, cudaStream_t stream);
// ---- attention_tc.cu : wgmma ViT attention (hd 64, non-causal, 129 <= S <= 257, exact full-row softmax) ----
bool attention_vit_tc_supported(int S);
int launch_attention_vit_tc(const bf16* qkv, bf16* out, int n_frames, int S, int H, int C, cudaStream_t stream);
int init_attention_tc_kernels();
// single-query attention against the cache at the decode positions above (kv_len = pos + 1):
// q [B, H*hd] -> o [B, H*hd], written in xwin layout with o_xwin. pages.table: a paged cache (kcache / vcache the
// layer's pool bases; clip b is cache slot b)
int launch_decode_attention(const bf16* q, long long q_ld, const bf16* kcache, const bf16* vcache,
                            bf16* o, long long o_ld, int B, int H, int head_dim, int s_max,
                            int kv_len, float scale, cudaStream_t stream, const int* pos_dev, bool o_xwin,
                            const int* n_pad, const KvPages& pages = KvPages());

// ---- decode_gemv.cu : decode-time weight streaming (1..64 new tokens) -------------------------------
// Two ring kernels (bulk-copy ring over a slot-ordered copy of the matrix + mma.sync) behind one launcher:
// 1..4 clips stage the activation vectors in shared memory (K <= 14336, optional fused RMSNorm and, for
// q|k|v, a fused token-embedding gather); 5..64 clips read activations that are already normalised
// and stored window-major ("xwin", below). Both read the copy that launch_gemv_repack builds, or its fp8 twin from
// launch_gemv_quantize_fp8 (E4M3 codes in the same order plus a power-of-two scale per row; decode_gemv.cu).
// per-CTA partial arg-max of the logits kernel: the next step's q|k|v kernel reduces the grid's
// partials itself (lowest index wins ties), so no arg-max kernel runs between two decode steps
struct ArgmaxPart { float v; int idx; };

struct GemvArgs {
  const bf16* x = nullptr; long long ldx = 0;   // [B][ldx] (5..64 clips: xwin layout, see below)
  const bf16* W_tiled = nullptr;                // slot-ordered copy of the [N, K] matrix ...
  const uint8_t* W_fp8 = nullptr;               // ... or its E4M3 codes in the same order (W_tiled null) with the
  const float* w_scale = nullptr;               //     row scales 2^e_r [N]: row r is W~[r] = code * 2^e_r
  int B = 0, N = 0, K = 0;
  const bf16* norm_w = nullptr; float eps = 0;  // 1..4 clips: optional fused RMSNorm prologue
  // 1..4 clips only. q|k|v with a fused token-embedding gather: x is row `token` of `embed` [vocab, K],
  // the token read from tok_in[b * tok_stride] or reduced from the previous step's arg-max partials
  // (amax_in [amax_n][B]); CTA 0 then stores the token (tok_out) and the raw row (h_out [B][K], the
  // residual stream). Logits: amax_out [gemv_grid(N)][B] receives the per-CTA partial arg-max.
  const bf16* embed = nullptr; int vocab = 0;
  const int* tok_in = nullptr; long long tok_stride = 0;
  const ArgmaxPart* amax_in = nullptr; int amax_n = 0;
  int* tok_out = nullptr; long long tok_out_stride = 0;
  bf16* h_out = nullptr;
  ArgmaxPart* amax_out = nullptr;
};

// what the projection's fused epilogue does with out[b][n] (the values are recorded by VCL_TC_TRACE)
enum GemvMode {
  GEMV_RES = 0,      // out[b, n] = bf16(bf16(x.W[n]) + res[b, n])   (res may alias out; res == null -> plain)
  GEMV_SWIGLU = 1,   // W rows interleaved (2j gate, 2j+1 up): out[b, j] = silu(gate)*up,  N = 2*F
  GEMV_QKV = 2,      // q|k|v projection + RoPE + cache write for one new token per clip, N = 3*H*128
  GEMV_LOGITS = 3    // logits (bf16-rounded, stored fp32) [B, N]; logits == null: only the arg-max partials
};
struct GemvEpilogue {
  int mode = GEMV_RES;
  bf16* out = nullptr; long long ldo = 0;       // RES: out[B][ldo]; SWIGLU: out[B][ldo] ...
  bool out_xwin = false;                        // ... or, 5..64 clips, in xwin layout (feeds down_proj)
  const bf16* res = nullptr; long long ldr = 0; // RES
  bf16* q_out = nullptr; long long ldq = 0;     // QKV: q [B][ldq], cache base of the layer [B][H][s_max][128]
  bf16* kcache = nullptr; bf16* vcache = nullptr;
  const bf16* cos_t = nullptr; const bf16* sin_t = nullptr;
  int H = 0, s_max = 0, pos = 0;
  const int* pos_dev = nullptr;                 // QKV: the decode positions above (pos_dev may be null) ...
  const int* n_pad = nullptr;                   // ... and the key floors [B] (required)
  KvPages pages;                                // QKV: a paged cache (kcache / vcache the layer's pool bases) or none
  float* logits = nullptr; long long ldl = 0;   // LOGITS
};

// xwin: element (b, k) of a [B][K] activation lives at xwin_offset(b, k, B); a buffer holds xwin_elems(B, K)
// elements
constexpr int XWIN_KC = 512, XWIN_PITCH = 544;        // 512 k per window row + 32 elements (64 B) of padding
__host__ __device__ inline size_t xwin_offset(int b, int k, int B) {
  return ((size_t)(k / XWIN_KC) * B + b) * XWIN_PITCH + (k % XWIN_KC);
}
inline size_t xwin_elems(int B, int K) { return (size_t)((K + XWIN_KC - 1) / XWIN_KC) * B * XWIN_PITCH; }
// y (xwin layout) = x [B][ldx] rows, RMS-normalised when w != null (LlamaRMSNorm rounding order)
int launch_xwin_norm(const bf16* x, long long ldx, bf16* y, const bf16* w, int B, int K, float eps, cudaStream_t stream);

int init_gemv_kernels();
// whether a [N, K] projection of B clips has a decode kernel. norm: with the fused RMSNorm (1..4 clips);
// 5..64 clips take any matrix whose K is a multiple of 32; fp8: the kernels of fp8 weights (their shared-memory
// plan; they take every shape the bf16 kernels take)
bool gemv_fits(int B, int N, int K, bool norm, bool fp8 = false);
int gemv_grid(int N);                         // CTAs of a 1..4-clip launch over N rows
size_t gemv_tiled_elems(int N, int K);        // elements of the slot-ordered copy of an [N, K] matrix
// qkv_pairs: rows are taken in the order of the fused q/k/v epilogue (RoPE pairs adjacent)
int launch_gemv_repack(const bf16* W, bf16* dst, int N, int K, bool qkv_pairs, cudaStream_t stream);
// The load-time E4M3 quantizer (rule: decode_gemv.cu, gemv_quantize_fp8_kernel). codes: gemv_tiled_elems(N, K)
// bytes in the slot order of launch_gemv_repack; scales [N] fp32 (2^e per row of that order); w_deq [N, K] bf16
// row-major receives W~ (may be W). bad (optional, device int[2], set to INT_MAX by the caller): the lowest
// source row with a non-finite weight, and the lowest whose W~ is not exactly a finite bf16 or whose scale is
// not a normal fp32 number.
int launch_gemv_quantize_fp8(const bf16* W, bf16* w_deq, uint8_t* codes, float* scales, int N, int K, bool qkv_pairs,
                             int* bad, cudaStream_t stream);
// 1..4 clips: gemv_tc_kernel; 5..64 clips: gemv_tcw_kernel with 1 / 2 / 4 clip groups at 5..16 / 17..32 / 33..64
// clips (row slices of at most 14 / 10 / 6 row groups per SM, for every epilogue)
int launch_gemv(const GemvArgs& a, const GemvEpilogue& e, cudaStream_t stream);

}  // namespace vcl

// C ABI of libvcl.so (declared in include/vcl.h): handle, weight repacking, and the launch
// sequences for the three stages of the hot path (SURVEY.md section 3.2):
//   vcl_clip_encode    CLIP ViT over the sampled frames
//   vcl_st_pool        spatio-temporal mean pool
//   vcl_llm_prefill / vcl_llm_decode_step / vcl_llm_generate   projector + splice + LLaMA
// Host code here only sequences kernels on the caller's stream; it never synchronises on the
// compute path and never touches a CPU implementation.
#include "../../include/vcl.h"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace vcl {

static thread_local char g_err[1024] = "";
static long long g_launches = 0;

// Every kernel launcher calls count_launches(1); graph replays add their node count.
void count_launches(long long n) { g_launches += n; }
long long launch_count() { return g_launches; }

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

}  // namespace vcl

using namespace vcl;

namespace {

struct ClipLayerW {
  bf16 *ln1_w, *ln1_b, *wqkv, *bqkv, *wo, *bo, *ln2_w, *ln2_b, *w1, *b1, *w2, *b2;
};
// The decode kernels' copy of one streamed matrix: bf16 slots, or E4M3 codes in the same order with a power-of-two
// scale per row (VCL_WEIGHTS_FP8_E4M3; decode_gemv.cu)
struct DecodeW {
  bf16* t = nullptr;
  uint8_t* q = nullptr;
  float* s = nullptr;
  void into(GemvArgs& g) const { g.W_tiled = t; g.W_fp8 = q; g.w_scale = s; }
};
struct LlmLayerW {
  bf16 *ln1, *wqkv, *wo, *ln2, *wgu, *wd;
  DecodeW qkv_d, o_d, gu_d, dn_d;   // slot-ordered copies for decode
};
struct GraphEntry {
  int B, n_new;        // the positions and pad counts are read on the device (h->d_pos, h->d_npad) ...
  int sampled;         // ... and so is the sampling table: a graph of the sampler serves every temperature / top_k /
                       // seed / top_n (h->sampler: 0 the arg-max, 1 the 16-bit sampler, 2 the 32-bit one, whose
                       // graphs serve every top_p / repetition penalty too)
  cudaGraphExec_t exec;
  long long kernels;   // kernel nodes in the graph (for vcl_launch_count)
  unsigned long long last_use;
};
constexpr size_t MAX_DECODE_GRAPHS = 6;   // LRU-bounded: an instantiated graph holds ~5 000 kernel nodes

// what one decode step reads and leaves behind
struct StepIo {
  const int32_t* tok_in = nullptr; long long in_stride = 1;      // the token fed at this step ...
  bool tok_from_partials = false;                                // ... or: the arg-max of the previous step's partials
  int32_t* tok_store = nullptr; long long store_stride = 1;      // where that reduced token is recorded
  bool partials_out = false;      // leave this step's arg-max as per-CTA partials for the next step (no arg-max kernel)
  float* logits_out = nullptr;
  int32_t* tok_out = nullptr; long long out_stride = 1;
  const int* pos_dev = nullptr;   // clip b at position pos + pos_dev[b] (null: pos)
  int sampled = 0;                // (h->sampler) the sampler picks tok_out (entry b of the sampling table for clip b) and writes
                                  // the log-probs of the entries that ask for them
};

// which sampling-table entries the rows of an lm_head call use, and the cache column their tokens take
// (SampleArgs in kernels.h; the counter subtracts the clip's left padding)
struct SampleAt {
  int on = 0;                                   // some entry samples or wants log-probs: the sampler replaces
                                                // the arg-max kernel (h->sampler: 2 the 32-bit sampler)
  int entry0 = 0; const int* rowmap = nullptr;  // row r: entry entry0 + (rowmap ? rowmap[r] : r)
  int col = 0; const int* col_dev = nullptr;    // row r: column col + (col_dev ? col_dev[r] : 0)
};

}  // namespace

struct vcl_handle {
  vcl_config cfg;
  int P = 0;         // patches per frame
  int KP = 0;        // padded im2col width
  int NV = 0;        // video tokens per clip = n_temporal + P
  std::vector<void*> allocs;
  bool clip_loaded = false, llm_loaded = false;
  // CLIP weights
  bf16 *patch_w = nullptr, *cls = nullptr, *pos = nullptr, *pre_w = nullptr, *pre_b = nullptr;
  std::vector<ClipLayerW> cl;
  // LLM weights
  bf16 *embed = nullptr, *norm_w = nullptr, *lm_head = nullptr;
  DecodeW lm_head_d;
  bf16 *proj_w0 = nullptr, *proj_b0 = nullptr, *proj_w1 = nullptr, *proj_b1 = nullptr;
  std::vector<LlmLayerW> ll;
  // CLIP activations (rows = max_frames * (P+1))
  bf16 *v_h = nullptr, *v_x = nullptr, *v_qkv = nullptr, *v_attn = nullptr, *v_act = nullptr;
  // LLM activations (rows = max_batch * max_seq)
  bf16 *l_h = nullptr, *l_x = nullptr, *l_qkv = nullptr, *l_attn = nullptr, *l_act = nullptr;
  bf16 *l_vid = nullptr, *l_vid_tmp = nullptr;
  bf16 *kcache = nullptr, *vcache = nullptr;   // [L][B][H][s_max][128]
  // the paged cache (cfg.kv_blocks > 0) instead: kv_blocks blocks of [L][K | V][H][128][128] (kernels.h: KvPages),
  // and the block table [n_slots_max()][table_row()] at a fixed device address, written whole from its host copy
  bf16* pool = nullptr;
  int* d_table = nullptr;
  std::vector<int> table_host;
  bf16 *rope_cos = nullptr, *rope_sin = nullptr;
  float* logits = nullptr;                     // [max_batch, vocab]
  int32_t* tokens = nullptr;                   // [max_batch, max_seq] generated-token scratch
  // decode activations ([max_batch, .])
  bf16 *d_h = nullptr, *d_x = nullptr, *d_q = nullptr, *d_qkv = nullptr, *d_attn = nullptr,
       *d_act = nullptr;
  std::vector<GraphEntry> graphs;
  unsigned long long graph_clock = 0;
  // The decode positions of kernels.h: a decode loop feeds clip b at d_pos[b] + step, with key floor d_npad[b].
  // Both arrays live at fixed addresses, so one captured decode graph per (B, n_new) serves every prompt
  // length, padding and set of slot positions. d_pos is written by each decode loop before it runs (the shared
  // prompt length, or one position per cache slot). d_npad holds the left padding of the cache
  // (vcl_llm_prefill_padded): the first d_npad[b] cache columns of clip b hold pad tokens. It is set by a padded
  // prefill, continued by appends and decode steps, and all zeros whenever the cache is not padded.
  int* d_pos = nullptr;                        // [max_batch]
  int* d_npad = nullptr;                       // [max_batch]
  bool padded = false;                         // host copies for the checks: d_npad is not all zeros ...
  int npad_max = 0;                            // ... and its largest entry
  ArgmaxPart* amax = nullptr;                  // [gemv_grid(vocab)][max_batch] per-CTA partial arg-max of the logits kernel
  int* d_pack = nullptr;                       // pack_elems(max_batch * max_seq): the packed-row map of kernels.h,
                                               // written by each vcl_llm_slots_prefill with one host-to-device copy
  // The sampling table (vcl_llm_set_sampling(_ex), vcl_llm_set_logprobs): entry b belongs to clip b / cache slot b.
  // One device block at a fixed address, [max_batch] seeds (u64), temperatures (f32), top_k (i32), top_n (i32),
  // top_p (f32), repetition penalties (f32), so one sampled decode graph serves every setting; samp_host is its host
  // copy, written whole by one host-to-device copy per call. Greedy without log-probs (top_n -1), top_p 1 and
  // penalty 1 at vcl_create.
  static constexpr int SAMP_BYTES = 28;   // per entry
  unsigned char* samp = nullptr;
  std::vector<unsigned char> samp_host;
  unsigned long long* samp_seed(unsigned char* base) const { return reinterpret_cast<unsigned long long*>(base); }
  float* samp_temp(unsigned char* base) const { return reinterpret_cast<float*>(base + 8 * cfg.max_batch); }
  int* samp_topk(unsigned char* base) const { return reinterpret_cast<int*>(base + 12 * cfg.max_batch); }
  int* samp_topn(unsigned char* base) const { return reinterpret_cast<int*>(base + 16 * cfg.max_batch); }
  float* samp_topp(unsigned char* base) const { return reinterpret_cast<float*>(base + 20 * cfg.max_batch); }
  float* samp_rep(unsigned char* base) const { return reinterpret_cast<float*>(base + 24 * cfg.max_batch); }
  // what entry b needs: 0 the arg-max, 1 the sampler (it samples, with a temperature above 0, or wants log-probs),
  // 2 the 32-bit sampler (a repetition penalty, or top-p on a sampled entry)
  int sampler_of(int b) {
    unsigned char* hb = samp_host.data();
    const float T = samp_temp(hb)[b];
    if (samp_rep(hb)[b] != 1.f || (T > 0.f && samp_topp(hb)[b] < 1.f)) return 2;
    return T > 0.f || samp_topn(hb)[b] >= 0 ? 1 : 0;
  }
  // ... and what entries first .. first + n - 1 need together
  int sampler(int first, int n) {
    int m = 0;
    for (int b = first; b < first + n; ++b) m = std::max(m, sampler_of(b));
    return m;
  }
  // The token sets of the repetition penalty (vcl_llm_set_token_set): a bitmap of tset_words() words per entry,
  // [max_batch][tset_words()], allocated by the first call that turns a penalty on or sets a token set
  unsigned int* tset = nullptr;
  int tset_words() const { return (cfg.vocab + 31) / 32; }
  // The log-prob buffer: two planes, int32 ids then f32 log-probs, each [max_batch][lp_rows()][1 + VCL_LOGPROBS_MAX],
  // indexed by entry and the RoPE position of the token (so a read is one contiguous copy per plane); allocated by the
  // first vcl_llm_set_logprobs that turns an entry on.
  unsigned char* lp = nullptr;
  int lp_rows() const { return cfg.max_seq + 1; }   // a decode loop's last token may take position max_seq
  size_t lp_plane() const { return (size_t)cfg.max_batch * lp_rows() * (1 + VCL_LOGPROBS_MAX); }   // elements

  size_t cache_layer_elems() const {
    return (size_t)cfg.max_batch * cfg.llm_heads * cfg.max_seq * 128;
  }
  bool paged() const { return cfg.kv_blocks > 0; }
  int table_row() const { return (cfg.max_seq + 127) / 128; }
  size_t block_elems() const { return (size_t)2 * cfg.llm_layers * cfg.llm_heads * 128 * 128; }
  KvPages pages() const {
    KvPages p;
    if (paged()) { p.table = d_table; p.row = table_row(); p.blk = (long long)block_elems(); }
    return p;
  }
  // rows of the LLM activations per clip: a paged handle prefills packed prompts, or chunks of longer prompts, of
  // at most 512 tokens only
  int act_seq() const { return paged() && cfg.max_seq > 512 ? 512 : cfg.max_seq; }
  // rows of the row-major lm_head: vocab rounded up to the 256-wide GEMM tile, the extra rows zero
  int vocab_padded() const { return (cfg.vocab + 255) / 256 * 256; }
  // cache slots: max_slots, or by default min(max_batch, 16)
  int n_slots_max() const { return cfg.max_slots > 0 ? cfg.max_slots : cfg.max_batch < 16 ? cfg.max_batch : 16; }
  // the capacity named in a slot-count rejection (the default's wording predates max_slots)
  std::string slots_note() const {
    char b[96];
    if (cfg.max_slots > 0) snprintf(b, sizeof b, "max_slots %d", cfg.max_slots);
    else snprintf(b, sizeof b, "max_batch %d, at most 16 slots", cfg.max_batch);
    return b;
  }
};

namespace {

template <class T>
int dalloc(vcl_handle* h, T** p, size_t n) {
  void* q = nullptr;
  cudaError_t e = cudaMalloc(&q, n * sizeof(T) + 256);
  if (e != cudaSuccess) {
    set_last_error("cudaMalloc of %zu bytes failed: %s", n * sizeof(T), cudaGetErrorString(e));
    return -2;
  }
  h->allocs.push_back(q);
  *p = reinterpret_cast<T*>(q);
  return 0;
}

typedef std::map<std::string, const vcl_tensor*> TensorMap;

const vcl_tensor* find_tensor(const TensorMap& m, const std::string& name, int ndim, long long d0,
                              long long d1 = -1, long long d2 = -1, long long d3 = -1) {
  auto it = m.find(name);
  if (it == m.end()) {
    set_last_error("missing weight '%s'", name.c_str());
    return nullptr;
  }
  const vcl_tensor* t = it->second;
  const long long want[4] = {d0, d1, d2, d3};
  bool ok = t->ndim == ndim && t->data != nullptr;
  for (int i = 0; ok && i < ndim; ++i) ok = (t->shape[i] == want[i]);
  if (!ok) {
    set_last_error("weight '%s' has shape [%lld,%lld,%lld,%lld] (ndim %d), expected [%lld,%lld,%lld,%lld] (ndim %d)",
                   name.c_str(), (long long)t->shape[0], (long long)t->shape[1],
                   (long long)t->shape[2], (long long)t->shape[3], t->ndim, d0, d1, d2, d3, ndim);
    return nullptr;
  }
  return t;
}

// allocate dst and copy a whole tensor
int load_copy(vcl_handle* h, const TensorMap& m, const std::string& name, bf16** dst, int ndim,
              long long d0, long long d1 = -1, long long d2 = -1, long long d3 = -1) {
  const vcl_tensor* t = find_tensor(m, name, ndim, d0, d1, d2, d3);
  if (!t) return -1;
  size_t n = 1;
  for (int i = 0; i < ndim; ++i) n *= (size_t)t->shape[i];
  if (dalloc(h, dst, n) != 0) return -2;
  VCL_CUDA_OK(cudaMemcpy(*dst, t->data, n * sizeof(bf16), cudaMemcpyDeviceToDevice));
  return 0;
}

int check_device() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_last_error("no CUDA device: %s (libvcl has no CPU fallback)", cudaGetErrorString(e));
    return -2;
  }
  int major = 0;
  VCL_CUDA_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  VCL_REQUIRE(major == 9, "device compute capability %d.x is not sm_90 (H100); libvcl is sm_90a only", major);
  return 0;
}

cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

#define VCL_TRY(expr)        \
  do {                       \
    int _rc = (expr);        \
    if (_rc != 0) return _rc; \
  } while (0)

int op_gemv_run(GemvArgs g, void* out, const void* res, float eps, cudaStream_t st);

// VCL_WEIGHTS_FP8_E4M3: every streamed matrix is quantized in place (W~ over the row-major copy, which the prefill
// GEMMs, the decode GEMM beyond 16 clips and the scoring lm_head read) and its decode copy is the E4M3 codes with
// one scale per row instead of the bf16 slots. The state-dict name of a failing matrix row is reported.
int quantize_llm_fp8(vcl_handle* h) {
  const vcl_config& c = h->cfg;
  const int D = c.llm_hidden, F = c.llm_inter, L = c.llm_layers, n_mats = 4 * L + 1;
  int* bad = nullptr;                                 // [n_mats][2] (see launch_gemv_quantize_fp8)
  VCL_CUDA_OK(cudaMalloc(&bad, (size_t)n_mats * 2 * sizeof(int)));
  VCL_CUDA_OK(cudaMemset(bad, 0x7f, (size_t)n_mats * 2 * sizeof(int)));
  auto quant = [&](bf16* W, DecodeW& d, int N, int K, bool qkv, int idx) -> int {
    if (dalloc(h, &d.q, gemv_tiled_elems(N, K)) || dalloc(h, &d.s, (size_t)N)) return -2;
    return launch_gemv_quantize_fp8(W, W, d.q, d.s, N, K, qkv, bad + 2 * idx, nullptr);
  };
  int rc = 0;
  for (int l = 0; l < L && rc == 0; ++l) {
    LlmLayerW& w = h->ll[l];
    rc = quant(w.wqkv, w.qkv_d, 3 * D, D, true, 4 * l);
    if (rc == 0) rc = quant(w.wo, w.o_d, D, D, false, 4 * l + 1);
    if (rc == 0) rc = quant(w.wgu, w.gu_d, 2 * F, D, false, 4 * l + 2);
    if (rc == 0) rc = quant(w.wd, w.dn_d, D, F, false, 4 * l + 3);
  }
  if (rc == 0) rc = quant(h->lm_head, h->lm_head_d, c.vocab, D, false, 4 * L);
  std::vector<int> flags((size_t)n_mats * 2);
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(flags.data(), bad, flags.size() * sizeof(int), cudaMemcpyDeviceToHost);
  cudaFree(bad);
  if (rc != 0) return rc;
  if (e != cudaSuccess) {
    set_last_error("vcl_load_llm_weights: %s", cudaGetErrorString(e));
    return -2;
  }
  // matrix idx, row r of its row-major (fused) layout -> the state-dict tensor and its row
  auto name_of = [&](int idx, int r, int* row) -> std::string {
    if (idx == 4 * L) { *row = r; return "lm_head.weight"; }
    const std::string lp = "model.layers." + std::to_string(idx / 4) + ".";
    switch (idx % 4) {
      case 0: { static const char* nm[3] = {"q_proj", "k_proj", "v_proj"};
                *row = r % D; return lp + "self_attn." + nm[r / D] + ".weight"; }
      case 1: *row = r; return lp + "self_attn.o_proj.weight";
      case 2: *row = r / 2; return lp + (r % 2 ? "mlp.up_proj.weight" : "mlp.gate_proj.weight");
      default: *row = r; return lp + "mlp.down_proj.weight";
    }
  };
  for (int idx = 0; idx < n_mats; ++idx) {
    int row = 0;
    if (flags[2 * idx] != 0x7f7f7f7f) {
      const std::string nm = name_of(idx, flags[2 * idx], &row);
      VCL_REQUIRE(false, "weight '%s' has a non-finite value in row %d: the fp8 weight format needs finite weights",
                  nm.c_str(), row);
    }
    if (flags[2 * idx + 1] != 0x7f7f7f7f) {
      const std::string nm = name_of(idx, flags[2 * idx + 1], &row);
      VCL_REQUIRE(false, "weight '%s' row %d: its fp8 row scale 2^e is not a normal fp32 number or its dequantized "
                  "values are not exact bf16 numbers (a row maximum below ~1e-36)", nm.c_str(), row);
    }
  }
  return 0;
}

}  // namespace

extern "C" {

int vcl_version(void) { return VCL_VERSION; }

const char* vcl_last_error(void) { return vcl::g_err; }

int vcl_create(vcl_handle** out, const vcl_config* c) {
  VCL_REQUIRE(out != nullptr && c != nullptr, "vcl_create: null argument");
  *out = nullptr;
  if (check_device() != 0) return -2;
  VCL_REQUIRE(c->clip_hidden > 0 && c->clip_heads > 0 && c->clip_hidden == c->clip_heads * 64,
              "vcl_create: CLIP head_dim must be 64 (hidden %d, heads %d)", c->clip_hidden, c->clip_heads);
  VCL_REQUIRE(c->clip_hidden % 256 == 0 && c->clip_inter % 256 == 0,
              "vcl_create: CLIP widths must be multiples of 256");
  VCL_REQUIRE(c->patch_size > 0 && c->image_size % c->patch_size == 0, "vcl_create: image/patch mismatch");
  VCL_REQUIRE(c->llm_hidden == c->llm_heads * 128, "vcl_create: LLM head_dim must be 128 (hidden %d, heads %d)",
              c->llm_hidden, c->llm_heads);
  VCL_REQUIRE(c->llm_hidden % 256 == 0 && c->llm_inter % 64 == 0, "vcl_create: LLM widths unsupported");
  VCL_REQUIRE(c->clip_layers >= 0 && c->llm_layers >= 0 && c->vocab > 0, "vcl_create: bad layer/vocab counts");
  VCL_REQUIRE(c->max_frames > 0 && c->max_batch > 0 && c->max_seq > 0, "vcl_create: capacities must be > 0");
  VCL_REQUIRE(c->proj_type == VCL_PROJ_LINEAR || c->proj_type == VCL_PROJ_MLP2X_GELU, "vcl_create: proj_type");
  VCL_REQUIRE(c->max_slots == 0 || (c->max_slots >= 1 && c->max_slots <= c->max_batch && c->max_slots <= 64),
              "vcl_create: max_slots=%d outside 1..%d (0: min(max_batch, 16))", c->max_slots,
              c->max_batch < 64 ? c->max_batch : 64);
  VCL_REQUIRE(c->kv_blocks == 0 || c->kv_blocks >= 2,
              "vcl_create: kv_blocks=%d: 0 (contiguous cache) or at least 2 (block 0 is the park block)", c->kv_blocks);
  {
    // every decode projection must have a kernel for every clip count up to 64 (beyond: the GEMM)
    const int D = c->llm_hidden, F = c->llm_inter;
    const struct { const char* name; int N, K; bool norm; } mats[5] = {
        {"q|k|v", 3 * D, D, true}, {"o_proj", D, D, false}, {"gate|up", 2 * F, D, true},
        {"down_proj", D, F, false}, {"lm_head", c->vocab, D, true}};
    for (int B = 1; B <= c->max_batch && B <= 64; ++B)
      for (const auto& m : mats)
        VCL_REQUIRE(gemv_fits(B, m.N, m.K, m.norm),
                    "vcl_create: the %s projection [%d x %d] has no decode kernel for %d clips (1..4 clips: K <= 14336 "
                    "and the shared-memory plan)", m.name, m.N, m.K, B);
  }

  vcl_handle* h = new vcl_handle();
  h->cfg = *c;
  const int G = c->image_size / c->patch_size;
  h->P = G * G;
  h->KP = ((3 * c->patch_size * c->patch_size + 63) / 64) * 64;
  h->NV = c->n_temporal + h->P;

  int rc = 0;
  rc |= init_gemm_kernels();
  rc |= init_attention_kernels();
  rc |= init_gemv_kernels();

  const size_t C = c->clip_hidden, F = c->clip_inter;
  const size_t Mv = (size_t)c->max_frames * (h->P + 1);
  const size_t act_elems = Mv * F > (size_t)c->max_frames * h->P * h->KP ? Mv * F
                                                                          : (size_t)c->max_frames * h->P * h->KP;
  rc |= dalloc(h, &h->v_h, Mv * C);
  rc |= dalloc(h, &h->v_x, Mv * C);
  rc |= dalloc(h, &h->v_qkv, Mv * 3 * C);
  rc |= dalloc(h, &h->v_attn, Mv * C);
  rc |= dalloc(h, &h->v_act, act_elems);

  const size_t D = c->llm_hidden, LF = c->llm_inter;
  const size_t Ml = (size_t)c->max_batch * h->act_seq();
  rc |= dalloc(h, &h->l_h, Ml * D);
  rc |= dalloc(h, &h->l_x, Ml * D);
  rc |= dalloc(h, &h->l_qkv, Ml * 3 * D);
  rc |= dalloc(h, &h->l_attn, Ml * D);
  rc |= dalloc(h, &h->l_act, Ml * LF);
  rc |= dalloc(h, &h->l_vid, (size_t)c->max_batch * h->NV * D);
  rc |= dalloc(h, &h->l_vid_tmp, (size_t)c->max_batch * h->NV * D);
  if (h->paged()) {
    rc |= dalloc(h, &h->pool, (size_t)c->kv_blocks * h->block_elems());
    h->table_host.assign((size_t)h->n_slots_max() * h->table_row(), 0);   // every entry at the park block
    rc |= dalloc(h, &h->d_table, h->table_host.size());
  } else {
    rc |= dalloc(h, &h->kcache, (size_t)c->llm_layers * h->cache_layer_elems());
    rc |= dalloc(h, &h->vcache, (size_t)c->llm_layers * h->cache_layer_elems());
  }
  rc |= dalloc(h, &h->rope_cos, (size_t)c->max_seq * 64);
  rc |= dalloc(h, &h->rope_sin, (size_t)c->max_seq * 64);
  rc |= dalloc(h, &h->logits, (size_t)c->max_batch * c->vocab);
  rc |= dalloc(h, &h->tokens, (size_t)c->max_batch * c->max_seq);
  const size_t Bm = c->max_batch;
  rc |= dalloc(h, &h->d_h, Bm * D);
  rc |= dalloc(h, &h->d_x, xwin_elems((int)Bm, (int)D) > Bm * D ? xwin_elems((int)Bm, (int)D) : Bm * D);
  rc |= dalloc(h, &h->d_q, Bm * D);
  rc |= dalloc(h, &h->d_qkv, Bm * 3 * D);
  rc |= dalloc(h, &h->d_attn, xwin_elems((int)Bm, (int)D) > Bm * D ? xwin_elems((int)Bm, (int)D) : Bm * D);
  rc |= dalloc(h, &h->d_act, xwin_elems((int)Bm, (int)LF) > Bm * LF ? xwin_elems((int)Bm, (int)LF) : Bm * LF);
  rc |= dalloc(h, &h->d_pos, Bm);
  rc |= dalloc(h, &h->d_npad, Bm);
  rc |= dalloc(h, &h->amax, (size_t)device_num_sms() * Bm);
  rc |= dalloc(h, &h->d_pack, pack_elems((long long)Ml));
  rc |= dalloc(h, &h->samp, Bm * vcl_handle::SAMP_BYTES);
  h->samp_host.assign(Bm * vcl_handle::SAMP_BYTES, 0);
  for (size_t b = 0; b < Bm; ++b) {
    h->samp_topn(h->samp_host.data())[b] = -1;
    h->samp_topp(h->samp_host.data())[b] = 1.f;
    h->samp_rep(h->samp_host.data())[b] = 1.f;
  }
  if (rc == 0) rc = launch_rope_table(h->rope_cos, h->rope_sin, c->max_seq, 128, c->rope_theta, 0);
  if (rc == 0) {
    cudaError_t e = cudaMemset(h->d_npad, 0, Bm * sizeof(int));   // the cache starts unpadded
    if (e == cudaSuccess)                                             // and every entry greedy, log-probs off
      e = cudaMemcpy(h->samp, h->samp_host.data(), h->samp_host.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && h->paged()) e = cudaMemset(h->d_table, 0, h->table_host.size() * sizeof(int));
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
      set_last_error("vcl_create: %s", cudaGetErrorString(e));
      rc = -2;
    }
  }
  if (rc != 0) {
    vcl_destroy(h);
    return -2;
  }
  *out = h;
  return 0;
}

void vcl_destroy(vcl_handle* h) {
  if (!h) return;
  for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
  for (void* p : h->allocs) cudaFree(p);
  delete h;
}

int vcl_load_clip_weights(vcl_handle* h, const vcl_tensor* tensors, int n) {
  VCL_REQUIRE(h && tensors && n > 0, "vcl_load_clip_weights: null argument");
  VCL_REQUIRE(!h->clip_loaded, "vcl_load_clip_weights: already loaded");
  TensorMap m;
  for (int i = 0; i < n; ++i)
    if (tensors[i].name) m[tensors[i].name] = &tensors[i];
  const vcl_config& c = h->cfg;
  const long long C = c.clip_hidden, F = c.clip_inter, ps = c.patch_size;
  const std::string pre = "vision_model.";
  // patch embedding [C,3,ps,ps] -> [C, KP] zero padded along K
  {
    const vcl_tensor* t = find_tensor(m, pre + "embeddings.patch_embedding.weight", 4, C, 3, ps, ps);
    if (!t) return -1;
    if (dalloc(h, &h->patch_w, (size_t)C * h->KP) != 0) return -2;
    VCL_CUDA_OK(cudaMemset(h->patch_w, 0, (size_t)C * h->KP * 2));
    const size_t k = 3 * ps * ps;
    VCL_CUDA_OK(cudaMemcpy2D(h->patch_w, (size_t)h->KP * 2, t->data, k * 2, k * 2, C,
                             cudaMemcpyDeviceToDevice));
  }
  if (load_copy(h, m, pre + "embeddings.class_embedding", &h->cls, 1, C)) return -1;
  if (load_copy(h, m, pre + "embeddings.position_embedding.weight", &h->pos, 2, h->P + 1, C)) return -1;
  if (load_copy(h, m, pre + "pre_layrnorm.weight", &h->pre_w, 1, C)) return -1;
  if (load_copy(h, m, pre + "pre_layrnorm.bias", &h->pre_b, 1, C)) return -1;
  h->cl.resize(c.clip_layers);
  for (int l = 0; l < c.clip_layers; ++l) {
    ClipLayerW& w = h->cl[l];
    const std::string lp = pre + "encoder.layers." + std::to_string(l) + ".";
    if (load_copy(h, m, lp + "layer_norm1.weight", &w.ln1_w, 1, C)) return -1;
    if (load_copy(h, m, lp + "layer_norm1.bias", &w.ln1_b, 1, C)) return -1;
    if (load_copy(h, m, lp + "layer_norm2.weight", &w.ln2_w, 1, C)) return -1;
    if (load_copy(h, m, lp + "layer_norm2.bias", &w.ln2_b, 1, C)) return -1;
    if (dalloc(h, &w.wqkv, (size_t)3 * C * C) || dalloc(h, &w.bqkv, (size_t)3 * C)) return -2;
    const char* nm[3] = {"q_proj", "k_proj", "v_proj"};
    for (int j = 0; j < 3; ++j) {
      const vcl_tensor* tw = find_tensor(m, lp + "self_attn." + nm[j] + ".weight", 2, C, C);
      const vcl_tensor* tb = find_tensor(m, lp + "self_attn." + nm[j] + ".bias", 1, C);
      if (!tw || !tb) return -1;
      VCL_CUDA_OK(cudaMemcpy(w.wqkv + (size_t)j * C * C, tw->data, (size_t)C * C * 2, cudaMemcpyDeviceToDevice));
      VCL_CUDA_OK(cudaMemcpy(w.bqkv + (size_t)j * C, tb->data, (size_t)C * 2, cudaMemcpyDeviceToDevice));
    }
    if (load_copy(h, m, lp + "self_attn.out_proj.weight", &w.wo, 2, C, C)) return -1;
    if (load_copy(h, m, lp + "self_attn.out_proj.bias", &w.bo, 1, C)) return -1;
    if (load_copy(h, m, lp + "mlp.fc1.weight", &w.w1, 2, F, C)) return -1;
    if (load_copy(h, m, lp + "mlp.fc1.bias", &w.b1, 1, F)) return -1;
    if (load_copy(h, m, lp + "mlp.fc2.weight", &w.w2, 2, C, F)) return -1;
    if (load_copy(h, m, lp + "mlp.fc2.bias", &w.b2, 1, C)) return -1;
  }
  VCL_CUDA_OK(cudaDeviceSynchronize());
  h->clip_loaded = true;
  return 0;
}

int vcl_load_llm_weights(vcl_handle* h, const vcl_tensor* tensors, int n) {
  return vcl_load_llm_weights_ex(h, tensors, n, VCL_WEIGHTS_BF16);
}

int vcl_load_llm_weights_ex(vcl_handle* h, const vcl_tensor* tensors, int n, int weight_format) {
  VCL_REQUIRE(weight_format == VCL_WEIGHTS_BF16 || weight_format == VCL_WEIGHTS_FP8_E4M3,
              "vcl_load_llm_weights: unknown weight format %d (VCL_WEIGHTS_BF16 0, VCL_WEIGHTS_FP8_E4M3 1)",
              weight_format);
  VCL_REQUIRE(h && tensors && n > 0, "vcl_load_llm_weights: null argument");
  VCL_REQUIRE(!h->llm_loaded, "vcl_load_llm_weights: already loaded");
  const bool fp8 = weight_format == VCL_WEIGHTS_FP8_E4M3;
  if (fp8) {
    // the fp8 decode kernels take every shape the bf16 ones take (vcl_create checked those)
    const vcl_config& c = h->cfg;
    const int D = c.llm_hidden, F = c.llm_inter;
    const struct { const char* name; int N, K; bool norm; } mats[5] = {
        {"q|k|v", 3 * D, D, true}, {"o_proj", D, D, false}, {"gate|up", 2 * F, D, true},
        {"down_proj", D, F, false}, {"lm_head", c.vocab, D, true}};
    for (int B = 1; B <= c.max_batch && B <= 64; ++B)
      for (const auto& mt : mats)
        VCL_REQUIRE(gemv_fits(B, mt.N, mt.K, mt.norm, true),
                    "vcl_load_llm_weights: the %s projection [%d x %d] has no fp8 decode kernel for %d clips", mt.name,
                    mt.N, mt.K, B);
  }
  TensorMap m;
  for (int i = 0; i < n; ++i)
    if (tensors[i].name) m[tensors[i].name] = &tensors[i];
  const vcl_config& c = h->cfg;
  const long long D = c.llm_hidden, F = c.llm_inter, V = c.vocab, CV = c.clip_hidden;
  if (load_copy(h, m, "model.embed_tokens.weight", &h->embed, 2, V, D)) return -1;
  if (load_copy(h, m, "model.norm.weight", &h->norm_w, 1, D)) return -1;
  {
    // row-major lm_head padded with zero rows to vocab_padded() (the scoring GEMM's N), decode reads the first V
    const vcl_tensor* t = find_tensor(m, "lm_head.weight", 2, V, D);
    if (!t) return -1;
    const size_t Vp = h->vocab_padded();
    if (dalloc(h, &h->lm_head, Vp * D) != 0) return -2;
    VCL_CUDA_OK(cudaMemset(h->lm_head + (size_t)V * D, 0, (Vp - V) * D * sizeof(bf16)));
    VCL_CUDA_OK(cudaMemcpy(h->lm_head, t->data, (size_t)V * D * sizeof(bf16), cudaMemcpyDeviceToDevice));
  }
  if (c.proj_type == VCL_PROJ_LINEAR) {
    if (load_copy(h, m, "model.mm_projector.weight", &h->proj_w0, 2, D, CV)) return -1;
    if (load_copy(h, m, "model.mm_projector.bias", &h->proj_b0, 1, D)) return -1;
  } else {
    if (load_copy(h, m, "model.mm_projector.0.weight", &h->proj_w0, 2, D, CV)) return -1;
    if (load_copy(h, m, "model.mm_projector.0.bias", &h->proj_b0, 1, D)) return -1;
    if (load_copy(h, m, "model.mm_projector.2.weight", &h->proj_w1, 2, D, D)) return -1;
    if (load_copy(h, m, "model.mm_projector.2.bias", &h->proj_b1, 1, D)) return -1;
  }
  h->ll.resize(c.llm_layers);
  for (int l = 0; l < c.llm_layers; ++l) {
    LlmLayerW& w = h->ll[l];
    const std::string lp = "model.layers." + std::to_string(l) + ".";
    if (load_copy(h, m, lp + "input_layernorm.weight", &w.ln1, 1, D)) return -1;
    if (load_copy(h, m, lp + "post_attention_layernorm.weight", &w.ln2, 1, D)) return -1;
    if (dalloc(h, &w.wqkv, (size_t)3 * D * D)) return -2;
    const char* nm[3] = {"q_proj", "k_proj", "v_proj"};
    for (int j = 0; j < 3; ++j) {
      const vcl_tensor* tw = find_tensor(m, lp + "self_attn." + nm[j] + ".weight", 2, D, D);
      if (!tw) return -1;
      VCL_CUDA_OK(cudaMemcpy(w.wqkv + (size_t)j * D * D, tw->data, (size_t)D * D * 2, cudaMemcpyDeviceToDevice));
    }
    if (load_copy(h, m, lp + "self_attn.o_proj.weight", &w.wo, 2, D, D)) return -1;
    // gate/up interleaved by row: row 2j = gate_j, row 2j+1 = up_j
    const vcl_tensor* tg = find_tensor(m, lp + "mlp.gate_proj.weight", 2, F, D);
    const vcl_tensor* tu = find_tensor(m, lp + "mlp.up_proj.weight", 2, F, D);
    if (!tg || !tu) return -1;
    if (dalloc(h, &w.wgu, (size_t)2 * F * D)) return -2;
    VCL_CUDA_OK(cudaMemcpy2D(w.wgu, (size_t)2 * D * 2, tg->data, (size_t)D * 2, (size_t)D * 2, F,
                             cudaMemcpyDeviceToDevice));
    VCL_CUDA_OK(cudaMemcpy2D(w.wgu + D, (size_t)2 * D * 2, tu->data, (size_t)D * 2, (size_t)D * 2, F,
                             cudaMemcpyDeviceToDevice));
    if (load_copy(h, m, lp + "mlp.down_proj.weight", &w.wd, 2, D, F)) return -1;
  }
  if (fp8) {
    VCL_TRY(quantize_llm_fp8(h));
    h->llm_loaded = true;
    return 0;
  }
  // Decode-only second copy of every streamed matrix in the slot order of the decode kernels (one bulk
  // copy per 16 KB slot, decode_gemv.cu). 13.2 GB more for the 7B model, 25.7 GB for 13B.
  auto tiled = [&](const bf16* src, DecodeW& dst, int N, int K, bool qkv) -> int {
    if (dalloc(h, &dst.t, gemv_tiled_elems(N, K))) return -2;
    return launch_gemv_repack(src, dst.t, N, K, qkv, nullptr);
  };
  for (int l = 0; l < c.llm_layers; ++l) {
    LlmLayerW& w = h->ll[l];
    if (tiled(w.wqkv, w.qkv_d, 3 * D, D, true) || tiled(w.wo, w.o_d, D, D, false) ||
        tiled(w.wgu, w.gu_d, 2 * F, D, false) || tiled(w.wd, w.dn_d, D, F, false)) return -2;
  }
  if (tiled(h->lm_head, h->lm_head_d, V, D, false)) return -2;
  VCL_CUDA_OK(cudaDeviceSynchronize());
  h->llm_loaded = true;
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// launch sequences
// ---------------------------------------------------------------------------------------------
namespace {

int gemm(const bf16* A, long long lda, const bf16* W, long long ldw, bf16* C, long long ldc,
         const bf16* bias, const bf16* res, long long ldr, int M, int N, int K, int act,
         cudaStream_t st, int block_n = 0, int cluster = 0) {
  GemmArgs g;
  g.cluster = cluster;
  g.A = A; g.lda = lda; g.W = W; g.ldw = ldw; g.C = C; g.ldc = ldc; g.bias = bias;
  g.residual = res; g.ldr = ldr; g.M = M; g.N = N; g.K = K; g.act = act; g.block_n = block_n;
  return launch_gemm_bf16_tn(g, st);
}

// CLIP ViT: leaves hidden_states[n_layers] in h->v_h ([n_frames, P+1, C])
int clip_forward(vcl_handle* h, const void* pixels, int fmt, int n_frames, int n_layers,
                 cudaStream_t st) {
  const vcl_config& c = h->cfg;
  VCL_REQUIRE(h->clip_loaded, "CLIP weights are not loaded");
  VCL_REQUIRE(n_frames > 0 && n_frames <= c.max_frames, "n_frames=%d outside 1..%d", n_frames, c.max_frames);
  VCL_REQUIRE(n_layers >= 0 && n_layers <= c.clip_layers, "n_layers=%d outside 0..%d", n_layers, c.clip_layers);
  VCL_REQUIRE(fmt == VCL_PIXELS_BF16_NCHW || fmt == VCL_PIXELS_U8_NHWC, "unknown pixel format %d", fmt);
  const int C = c.clip_hidden, F = c.clip_inter, P = h->P, S = P + 1;
  const int M = n_frames * S;
  bf16* patchA = h->v_act;      // [n_frames*P, KP]   (aliases the MLP buffer, dead before layer 0)
  bf16* patch_out = h->v_qkv;   // [n_frames*P, C]
  VCL_TRY(launch_im2col(pixels, fmt, patchA, n_frames, c.image_size, c.patch_size, h->KP, st));
  VCL_TRY(gemm(patchA, h->KP, h->patch_w, h->KP, patch_out, C, nullptr, nullptr, 0, n_frames * P, C,
               h->KP, ACT_NONE, st));
  VCL_TRY(launch_clip_embed_ln(patch_out, h->cls, h->pos, h->pre_w, h->pre_b, h->v_h, n_frames, P, C,
                               c.clip_ln_eps, st));
  for (int l = 0; l < n_layers; ++l) {
    const ClipLayerW& w = h->cl[l];
    VCL_TRY(launch_layernorm(h->v_h, C, h->v_x, C, w.ln1_w, w.ln1_b, M, C, c.clip_ln_eps, st));
    VCL_TRY(gemm(h->v_x, C, w.wqkv, C, h->v_qkv, 3 * C, w.bqkv, nullptr, 0, M, 3 * C, C, ACT_NONE, st));
    VCL_TRY(launch_attention_vit(h->v_qkv, h->v_attn, n_frames, S, c.clip_heads, C, st));
    VCL_TRY(gemm(h->v_attn, C, w.wo, C, h->v_h, C, w.bo, h->v_h, C, M, C, C, ACT_NONE, st));
    VCL_TRY(launch_layernorm(h->v_h, C, h->v_x, C, w.ln2_w, w.ln2_b, M, C, c.clip_ln_eps, st));
    VCL_TRY(gemm(h->v_x, C, w.w1, C, h->v_act, F, w.b1, nullptr, 0, M, F, C, ACT_QGELU, st));
    VCL_TRY(gemm(h->v_act, F, w.w2, F, h->v_h, C, w.b2, h->v_h, C, M, C, F, ACT_NONE, st));
  }
  return 0;
}

// the K / V cache base of layer l: its contiguous cache, or in a paged cache its place inside block 0 (h->pages()
// adds the block offset of a column)
bf16* kc_layer(vcl_handle* h, int l) {
  if (h->paged()) return h->pool + (size_t)(2 * l) * h->cfg.llm_heads * 128 * 128;
  return h->kcache + (size_t)l * h->cache_layer_elems();
}
bf16* vc_layer(vcl_handle* h, int l) {
  if (h->paged()) return h->pool + (size_t)(2 * l + 1) * h->cfg.llm_heads * 128 * 128;
  return h->vcache + (size_t)l * h->cache_layer_elems();
}

// the static entry points: a paged cache serves the slot entry points only
#define VCL_NOT_PAGED(h, name)                                                                                   \
  VCL_REQUIRE(!(h)->paged(), "%s: this handle has a paged KV cache (kv_blocks %d), which serves the slot entry "   \
              "points only (generate_requests: vcl_llm_slots_prefill / vcl_llm_slot_prefill / vcl_llm_slot_decode)", \
              name, (h)->cfg.kv_blocks)

// final RMSNorm + lm_head on rows x[b*ldx .. ] (b < B), arg-max
// partials_out: the arg-max is left as per-CTA partials in h->amax for the next step's q|k|v kernel
// smp.on: the sampler picks the tokens instead of the arg-max kernel (the logits are then always written)
int lm_head_argmax(vcl_handle* h, const bf16* x, long long ldx, int B, float* logits_out,
                   int32_t* tok_out, long long tok_stride, cudaStream_t st, bool partials_out = false,
                   const SampleAt& smp = SampleAt()) {
  const vcl_config& c = h->cfg;
  VCL_REQUIRE(!(partials_out && smp.on), "sampled rows need the logits, not the partial arg-max");
  GemvArgs g;
  h->lm_head_d.into(g); g.N = c.vocab; g.K = c.llm_hidden;
  GemvEpilogue e;
  e.mode = GEMV_LOGITS; e.ldl = c.vocab;
  if (B <= 4) {
    g.x = x; g.ldx = ldx; g.B = B; g.norm_w = h->norm_w; g.eps = c.rms_eps;
    if (partials_out) {
      g.amax_out = h->amax;
      return launch_gemv(g, e, st);
    }
    e.logits = h->logits;
    VCL_TRY(launch_gemv(g, e, st));
  } else if (B <= 64) {
    // 5..64 clips: the rows normalised into the window-major layout first, then one ring kernel over the
    // vocabulary matrix (in row slices)
    g.x = h->d_x; g.ldx = c.llm_hidden; g.B = B;
    VCL_TRY(launch_xwin_norm(x, ldx, h->d_x, h->norm_w, B, c.llm_hidden, c.rms_eps, st));
    e.logits = h->logits;
    VCL_TRY(launch_gemv(g, e, st));
  } else {
    // more than 64 rows are split into ceil(B / 16) near-equal chunks of the 5..16-clip kernel
    const int n_chunks = (B + 15) / 16;
    for (int i = 0; i < n_chunks; ++i) {
      const int b0 = B * i / n_chunks, nb = B * (i + 1) / n_chunks - b0;
      g.x = h->d_x; g.ldx = c.llm_hidden; g.B = nb;
      VCL_TRY(launch_xwin_norm(x + (long long)b0 * ldx, ldx, h->d_x, h->norm_w, nb, c.llm_hidden, c.rms_eps, st));
      e.logits = h->logits + (size_t)b0 * c.vocab;
      VCL_TRY(launch_gemv(g, e, st));
    }
  }
  if (logits_out != nullptr && logits_out != h->logits)
    VCL_CUDA_OK(cudaMemcpyAsync(logits_out, h->logits, (size_t)B * c.vocab * sizeof(float),
                                cudaMemcpyDeviceToDevice, st));
  if (tok_out != nullptr && smp.on) {
    SampleArgs sa;
    sa.logits = h->logits; sa.ld = c.vocab; sa.V = c.vocab; sa.B = B;
    sa.temperature = h->samp_temp(h->samp); sa.top_k = h->samp_topk(h->samp); sa.seed = h->samp_seed(h->samp);
    sa.entry0 = smp.entry0; sa.rowmap = smp.rowmap; sa.col = smp.col; sa.col_dev = smp.col_dev; sa.n_pad = h->d_npad;
    sa.out = tok_out; sa.out_stride = tok_stride;
    if (h->lp != nullptr) {   // (every top_n entry is -1 until the buffer exists)
      sa.top_n = h->samp_topn(h->samp);
      sa.lp_id = reinterpret_cast<int*>(h->lp); sa.lp_val = reinterpret_cast<float*>(h->lp) + h->lp_plane();
      sa.lp_entry = (long long)h->lp_rows() * (1 + VCL_LOGPROBS_MAX); sa.lp_pos = 1 + VCL_LOGPROBS_MAX;
      sa.lp_rows = h->lp_rows();
    }
    if (smp.on == 2) {   // the 32-bit sampler: top_p, the penalties and the token sets
      sa.top_p = h->samp_topp(h->samp); sa.rep = h->samp_rep(h->samp);
      sa.tset = h->tset; sa.tset_words = h->tset_words();
    }
    return launch_sample(sa, st);
  }
  if (tok_out != nullptr) VCL_TRY(launch_argmax(h->logits, tok_out, tok_stride, B, c.vocab, st));
  return 0;
}

// start_pos > 0 continues a cached sequence: the S new tokens take positions start_pos .. start_pos+S-1
// and attend to the whole cache (multi-turn reuse; no video span in a continuation).
// states_out (optional): [n_layers + 1][B][S][D], entry i = HF's hidden_states[i] (the raw output of
// layer i; entry 0 the spliced input embeddings), copied out as the stack advances.
// A new sequence (start_pos == 0) sets the cache's left padding: n_pad_host [B] (host memory), or none when it is
// null or all zero. A continuation keeps the padding of the cache.
// slot > 0 (B = 1): the sequence goes to clip `slot` of the cache; every layer's cache base moves by that many
// clips, and no other clip's columns are read or written.
// packed_rows > 0: B new sequences packed without padding into packed_rows rows, each into its own cache slot, as
// the map in h->d_pack (kernels.h) describes them; S is the longest. Every row is computed as it would be in a
// prefill of its sequence alone; next_tok [B] receives each sequence's first token. pack_attn: which packed
// attention kernels run (1: wgmma, the sequences with pack_len > 0; 2: flash, chunks of longer prompts; 3: both).
int llm_prefill(vcl_handle* h, const int64_t* ids, const void* video_feats, const int32_t* vid_start,
                int B, int S, int n_layers, void* hidden_out, float* logits_out, int32_t* next_tok,
                long long tok_stride, cudaStream_t st, int start_pos = 0, void* states_out = nullptr,
                const int32_t* n_pad_host = nullptr, int slot = 0, int packed_rows = 0, int pack_sampled = 0,
                int pack_attn = 1) {
  const vcl_config& c = h->cfg;
  const bool packed = packed_rows > 0;
  VCL_REQUIRE(h->llm_loaded, "LLM weights are not loaded");
  VCL_REQUIRE(packed || !h->paged(), "a paged KV cache is prefilled by packed prefills only");
  VCL_REQUIRE(B > 0 && B <= c.max_batch, "B=%d outside 1..%d", B, c.max_batch);
  VCL_REQUIRE(slot == 0 || (B == 1 && slot > 0 && slot < c.max_batch), "slot %d needs B = 1 and a clip of the cache",
              slot);
  VCL_REQUIRE(!packed || (start_pos == 0 && n_pad_host == nullptr && states_out == nullptr && hidden_out == nullptr &&
                          logits_out == nullptr && slot == 0),
              "packed sequences start unpadded and return their next tokens only");
  VCL_REQUIRE(S > 0 && start_pos >= 0 && start_pos + S <= c.max_seq, "positions %d..%d outside the cache (max_seq %d)",
              start_pos, start_pos + S - 1, c.max_seq);
  VCL_REQUIRE(n_layers >= 0 && n_layers <= c.llm_layers, "n_layers=%d outside 0..%d", n_layers, c.llm_layers);
  VCL_REQUIRE(ids != nullptr && (vid_start != nullptr || start_pos > 0 || (packed && video_feats == nullptr)),
              "ids / vid_start are required");
  VCL_REQUIRE(start_pos == 0 || video_feats == nullptr, "a continuation cannot carry a video span");
  VCL_REQUIRE((logits_out == nullptr && next_tok == nullptr) || n_layers == c.llm_layers,
              "logits / next token need the full stack (n_layers == %d)", c.llm_layers);
  if (start_pos == 0) {
    int npad_max = 0;
    if (n_pad_host != nullptr) {
      for (int b = 0; b < B; ++b) {
        VCL_REQUIRE(n_pad_host[b] >= 0 && n_pad_host[b] < S,
                    "n_pad[%d] = %d outside 0..%d (a row needs at least one real token)", b, n_pad_host[b], S - 1);
        npad_max = n_pad_host[b] > npad_max ? n_pad_host[b] : npad_max;
      }
    }
    if (npad_max > 0)
      VCL_CUDA_OK(cudaMemcpyAsync(h->d_npad, n_pad_host, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    else if (h->padded)
      VCL_CUDA_OK(cudaMemsetAsync(h->d_npad, 0, (size_t)c.max_batch * sizeof(int32_t), st));
    h->padded = npad_max > 0;
    h->npad_max = npad_max;
  } else {
    VCL_REQUIRE(start_pos > h->npad_max, "start_pos %d lies inside the left padding (%d columns)", start_pos,
                h->npad_max);
  }
  const int* np = h->padded ? h->d_npad : nullptr;
  const int* pk = packed ? h->d_pack : nullptr;
  const int D = c.llm_hidden, F = c.llm_inter, H = c.llm_heads, NV = h->NV;
  const int M = packed ? packed_rows : B * S;
  const size_t slot_off = (size_t)slot * H * c.max_seq * 128;
  auto kc = [&](int l) { return kc_layer(h, l) + slot_off; };
  auto vc = [&](int l) { return vc_layer(h, l) + slot_off; };
  if (video_feats != nullptr) {
    const bf16* vf = reinterpret_cast<const bf16*>(video_feats);
    if (c.proj_type == VCL_PROJ_LINEAR) {
      VCL_TRY(gemm(vf, c.clip_hidden, h->proj_w0, c.clip_hidden, h->l_vid, D, h->proj_b0, nullptr, 0,
                   B * NV, D, c.clip_hidden, ACT_NONE, st));
    } else {
      VCL_TRY(gemm(vf, c.clip_hidden, h->proj_w0, c.clip_hidden, h->l_vid_tmp, D, h->proj_b0, nullptr, 0,
                   B * NV, D, c.clip_hidden, ACT_GELU, st));
      VCL_TRY(gemm(h->l_vid_tmp, D, h->proj_w1, D, h->l_vid, D, h->proj_b1, nullptr, 0, B * NV, D, D,
                   ACT_NONE, st));
    }
  }
  VCL_TRY(launch_embed_splice(reinterpret_cast<const long long*>(ids), h->embed, h->l_vid, vid_start,
                              h->l_h, B, S, D, video_feats ? NV : 0, c.vocab, st, pk, M));
  const float scale = 0.08838834764831845f;  // 128 ^ -1/2
  auto keep_state = [&](int i) -> int {
    if (states_out == nullptr) return 0;
    VCL_CUDA_OK(cudaMemcpyAsync(reinterpret_cast<bf16*>(states_out) + (size_t)i * M * D, h->l_h, (size_t)M * D * 2,
                                cudaMemcpyDeviceToDevice, st));
    return 0;
  };
  VCL_TRY(keep_state(0));
  for (int l = 0; l < n_layers; ++l) {
    const LlmLayerW& w = h->ll[l];
    VCL_TRY(launch_rmsnorm(h->l_h, D, h->l_x, D, w.ln1, M, D, c.rms_eps, st));
    // q|k|v projection with RoPE and the KV-cache write in its epilogue: q lands (rotated) in l_qkv, k and v in
    // the cache. VCL_PREFILL_ROPE_SEPARATE=1: plain GEMM + rope_kv_prefill_kernel (A/B; packed sequences always
    // take the epilogue)
    static const bool rope_separate = getenv("VCL_PREFILL_ROPE_SEPARATE") != nullptr;
    if (!rope_separate || packed) {
      GemmArgs g;
      g.A = h->l_x; g.lda = D; g.W = w.wqkv; g.ldw = D; g.C = h->l_qkv; g.ldc = 3 * D; g.M = M; g.N = 3 * D; g.K = D;
      g.act = ACT_ROPE;
      g.rope.cos_t = h->rope_cos; g.rope.sin_t = h->rope_sin; g.rope.kcache = kc(l); g.rope.vcache = vc(l);
      g.rope.S = S; g.rope.start_pos = start_pos; g.rope.H = H; g.rope.s_max = c.max_seq; g.rope.n_pad = np;
      g.rope.pack = pk; g.rope.pages = h->pages();
      VCL_TRY(launch_gemm_bf16_tn(g, st));
    } else {
      VCL_TRY(gemm(h->l_x, D, w.wqkv, D, h->l_qkv, 3 * D, nullptr, nullptr, 0, M, 3 * D, D, ACT_NONE, st));
      VCL_TRY(launch_rope_kv_prefill(h->l_qkv, kc(l), vc(l), h->rope_cos, h->rope_sin, B,
                                     S, H, 128, c.max_seq, start_pos, st, nullptr, np));
    }
    AttnArgs a;
    a.q = h->l_qkv; a.q_sb = (long long)S * 3 * D; a.q_sh = 128; a.q_ss = 3 * D;
    a.k = kc(l); a.k_sb = (long long)H * c.max_seq * 128; a.k_sh = (long long)c.max_seq * 128; a.k_ss = 128;
    a.v = vc(l); a.v_sb = a.k_sb; a.v_sh = a.k_sh; a.v_ss = 128;
    a.o = h->l_attn; a.o_sb = (long long)S * D; a.o_sh = 128; a.o_ss = D;
    a.B = B; a.H = H; a.S = S; a.head_dim = 128; a.scale = scale; a.causal = 1;
    a.S_kv = start_pos + S; a.q_off = start_pos; a.n_pad = np; a.pack = pk;
    if (h->paged()) {   // heads 128 x 128 apart inside a block (kernels.h: KvPages)
      a.k_sb = a.v_sb = 0; a.k_sh = a.v_sh = 128 * 128; a.pages = h->pages();
      a.pack_tc = (pack_attn & 1) != 0; a.pack_flash = (pack_attn & 2) != 0;
    }
    VCL_TRY(launch_attention(a, st));
    VCL_TRY(gemm(h->l_attn, D, w.wo, D, h->l_h, D, nullptr, h->l_h, D, M, D, D, ACT_NONE, st));
    VCL_TRY(launch_rmsnorm(h->l_h, D, h->l_x, D, w.ln2, M, D, c.rms_eps, st));
    VCL_TRY(gemm(h->l_x, D, w.wgu, D, h->l_act, F, nullptr, nullptr, 0, M, 2 * F, D, ACT_SWIGLU, st));
    VCL_TRY(gemm(h->l_act, F, w.wd, F, h->l_h, D, nullptr, h->l_h, D, M, D, F, ACT_NONE, st));
    VCL_TRY(keep_state(l + 1));
  }
  if (hidden_out != nullptr)
    VCL_CUDA_OK(cudaMemcpyAsync(hidden_out, h->l_h, (size_t)M * D * 2, cudaMemcpyDeviceToDevice, st));
  if (packed && next_tok != nullptr) {
    // each sequence's last row, gathered into B contiguous rows of l_x (dead after the last layer)
    VCL_TRY(launch_embed_tokens(pack_last(pk), 1, h->l_h, h->l_x, B, D, M, st));
    // sequence i samples with its slot's entry; its token takes column start_i + S_i
    SampleAt smp;
    smp.on = pack_sampled; smp.rowmap = pack_slot(pk); smp.col_dev = pack_end(pk);
    return lm_head_argmax(h, h->l_x, D, B, nullptr, next_tok, tok_stride, st, false, smp);
  }
  if (logits_out != nullptr || next_tok != nullptr) {
    SampleAt smp;   // clip b (slot `slot` for B = 1) samples with its entry; its token takes column start_pos + S
    smp.on = next_tok != nullptr ? h->sampler(slot, B) : 0; smp.entry0 = slot; smp.col = start_pos + S;
    VCL_TRY(lm_head_argmax(h, h->l_h + (size_t)(S - 1) * D, (long long)S * D, B, logits_out, next_tok,
                           tok_stride, st, false, smp));
  }
  return 0;
}

// Rows per lm_head GEMM of the scoring tail: as many [., vocab_padded] bf16 rows as the q|k|v activation
// (max_batch * max_seq * 3D elements) holds, in whole 128-row tiles when there is room for one.
int score_chunk_rows(const vcl_handle* h) {
  const long long cap = (long long)h->cfg.max_batch * h->cfg.max_seq * 3 * h->cfg.llm_hidden / h->vocab_padded();
  return (int)(cap >= 128 ? cap / 128 * 128 : cap);
}

// Scoring tail after a full-depth prefill (h->l_h: the last layer's output, B*S rows): the final RMSNorm over
// every row into l_x, then per chunk of rows the lm_head GEMM into l_qkv (dead after the last layer) and the
// cross-entropy kernel over it. The per-row NLL waits in l_attn (also dead) for the mean over all rows. The KV
// cache is not touched. labels [B,S] (HF's shift: column s is scored against labels[b, s+1]) or null.
int score_tail(vcl_handle* h, int B, int S, const int64_t* labels, bf16* logits_out, float* nll_out,
               float* loss_out, cudaStream_t st) {
  const vcl_config& c = h->cfg;
  const int D = c.llm_hidden, V = c.vocab, Vp = h->vocab_padded();
  const long long M = (long long)B * S;
  const int chunk = score_chunk_rows(h);
  VCL_REQUIRE(chunk > 0, "scoring needs max_batch * max_seq * 3 * llm_hidden >= %d (one padded vocabulary row)", Vp);
  const long long* lab = reinterpret_cast<const long long*>(labels);
  float* nll = labels != nullptr ? reinterpret_cast<float*>(h->l_attn) : nullptr;
  VCL_TRY(launch_rmsnorm(h->l_h, D, h->l_x, D, h->norm_w, (int)M, D, c.rms_eps, st));
  for (long long r0 = 0; r0 < M; r0 += chunk) {
    const int m = (int)(M - r0 < chunk ? M - r0 : chunk);
    VCL_TRY(gemm(h->l_x + r0 * D, D, h->lm_head, D, h->l_qkv, Vp, nullptr, nullptr, 0, m, Vp, D, ACT_NONE, st));
    VCL_TRY(launch_cross_entropy(h->l_qkv, Vp, V, lab, r0, m, S, nll != nullptr ? nll + r0 : nullptr,
                                 logits_out != nullptr ? logits_out + r0 * V : nullptr, st));
  }
  if (labels != nullptr) VCL_TRY(launch_nll_mean(nll, lab, M, S, nll_out, loss_out, st));
  return 0;
}

// One decode step: the token of io is fed to clip b at position pos (+ io.pos_dev[b]), key floor h->d_npad[b].
int llm_decode_step(vcl_handle* h, const StepIo& io, int B, int pos, cudaStream_t st) {
  const vcl_config& c = h->cfg;
  const int D = c.llm_hidden, F = c.llm_inter, H = c.llm_heads;
  const float scale = 0.08838834764831845f;
  const int* pd = io.pos_dev;
  const int* np = h->d_npad;
  VCL_REQUIRE(pos >= 0 && pos < c.max_seq, "decode position %d outside the cache (max_seq %d)", pos, c.max_seq);
  VCL_REQUIRE(pd != nullptr || pos >= h->npad_max, "decode position %d lies inside the left padding (%d columns)",
              pos, h->npad_max);
  // 1..4 clips: the embedding lookup is part of layer 0's q|k|v kernel (and with it the arg-max of the
  // previous step); every other path gathers the rows with a kernel of its own.
  const bool fused_embed = B <= 4 && c.llm_layers > 0;
  VCL_REQUIRE(fused_embed || (!io.tok_from_partials && !io.partials_out), "partial arg-max hand-off needs 1..4 clips");
  if (!fused_embed) VCL_TRY(launch_embed_tokens(io.tok_in, io.in_stride, h->embed, h->d_h, B, D, c.vocab, st));
  for (int l = 0; l < c.llm_layers; ++l) {
    const LlmLayerW& w = h->ll[l];
    if (B <= 64) {
      // the ring kernels. 1..4 clips fuse the RMSNorm into the projection (and, in layer 0, the embedding
      // gather); 5..64 clips take their inputs window-major (kernels.h: xwin), written by launch_xwin_norm,
      // the attention kernel and the SwiGLU epilogue. The residual stream d_h stays row-major.
      const bool wide = B > 4;
      auto normed = [&](GemvArgs& g, const bf16* ln) -> int {
        g.ldx = D;
        if (wide) {
          g.x = h->d_x;
          return launch_xwin_norm(h->d_h, D, h->d_x, ln, B, D, c.rms_eps, st);
        }
        g.x = h->d_h; g.norm_w = ln; g.eps = c.rms_eps;
        return 0;
      };
      GemvEpilogue residual;
      residual.mode = GEMV_RES; residual.out = h->d_h; residual.ldo = D; residual.res = h->d_h; residual.ldr = D;

      GemvArgs g;
      w.qkv_d.into(g); g.B = B; g.N = 3 * D; g.K = D;
      VCL_TRY(normed(g, w.ln1));
      if (fused_embed && l == 0) {
        g.x = nullptr; g.embed = h->embed; g.vocab = c.vocab; g.h_out = h->d_h;
        if (io.tok_from_partials) {
          g.amax_in = h->amax; g.amax_n = gemv_grid(c.vocab); g.tok_out = io.tok_store; g.tok_out_stride = io.store_stride;
        } else {
          g.tok_in = io.tok_in; g.tok_stride = io.in_stride;
        }
      }
      GemvEpilogue qkv;
      qkv.mode = GEMV_QKV; qkv.q_out = h->d_q; qkv.ldq = D; qkv.kcache = kc_layer(h, l); qkv.vcache = vc_layer(h, l);
      qkv.cos_t = h->rope_cos; qkv.sin_t = h->rope_sin; qkv.H = H; qkv.s_max = c.max_seq; qkv.pos = pos; qkv.pos_dev = pd;
      qkv.n_pad = np; qkv.pages = h->pages();
      VCL_TRY(launch_gemv(g, qkv, st));
      VCL_TRY(launch_decode_attention(h->d_q, D, kc_layer(h, l), vc_layer(h, l), h->d_attn, D, B, H, 128,
                                      c.max_seq, pos + 1, scale, st, pd, /*o_xwin=*/wide, np, h->pages()));
      GemvArgs go;
      go.x = h->d_attn; go.ldx = D; w.o_d.into(go); go.B = B; go.N = D; go.K = D;
      VCL_TRY(launch_gemv(go, residual, st));
      GemvArgs gg;
      w.gu_d.into(gg); gg.B = B; gg.N = 2 * F; gg.K = D;
      VCL_TRY(normed(gg, w.ln2));
      GemvEpilogue swiglu;
      swiglu.mode = GEMV_SWIGLU; swiglu.out = h->d_act; swiglu.ldo = F; swiglu.out_xwin = wide;
      VCL_TRY(launch_gemv(gg, swiglu, st));
      GemvArgs gd;
      gd.x = h->d_act; gd.ldx = F; w.dn_d.into(gd); gd.B = B; gd.N = D; gd.K = F;
      VCL_TRY(launch_gemv(gd, residual, st));
    } else {
      // B > 64: tensor-core path, the B new rows ride in one (mostly empty) 128-row tile and the
      // N tile is narrowed so that every SM streams a slice of the weights
      VCL_REQUIRE(!h->paged(), "a paged KV cache decodes at most 64 slots");
      VCL_TRY(launch_rmsnorm(h->d_h, D, h->d_x, D, w.ln1, B, D, c.rms_eps, st));
      VCL_TRY(gemm(h->d_x, D, w.wqkv, D, h->d_qkv, 3 * D, nullptr, nullptr, 0, B, 3 * D, D, ACT_NONE, st));
      VCL_TRY(launch_rope_kv_prefill(h->d_qkv, kc_layer(h, l), vc_layer(h, l), h->rope_cos, h->rope_sin, B,
                                     1, H, 128, c.max_seq, pos, st, pd, np));
      VCL_TRY(launch_decode_attention(h->d_qkv, 3 * D, kc_layer(h, l), vc_layer(h, l), h->d_attn, D, B, H,
                                      128, c.max_seq, pos + 1, scale, st, pd, false, np));
      VCL_TRY(gemm(h->d_attn, D, w.wo, D, h->d_h, D, nullptr, h->d_h, D, B, D, D, ACT_NONE, st));
      VCL_TRY(launch_rmsnorm(h->d_h, D, h->d_x, D, w.ln2, B, D, c.rms_eps, st));
      VCL_TRY(gemm(h->d_x, D, w.wgu, D, h->d_act, F, nullptr, nullptr, 0, B, 2 * F, D, ACT_SWIGLU, st));
      VCL_TRY(gemm(h->d_act, F, w.wd, F, h->d_h, D, nullptr, h->d_h, D, B, D, F, ACT_NONE, st));
    }
  }
  SampleAt smp;   // the token fed at column c_b is followed by one at column c_b + 1
  smp.on = io.sampled; smp.col = pos + 1; smp.col_dev = pd;
  VCL_TRY(lm_head_argmax(h, h->d_h, D, B, io.logits_out, io.tok_out, io.out_stride, st, io.partials_out, smp));
  return 0;
}

// Steps 1 .. n_new-1 of a greedy loop over the token scratch tk [B][n_new] (tk[:, 0] is given).
// For 1..4 clips no arg-max / embedding kernel runs between two steps: the logits kernel leaves
// per-CTA partials, the next step's first q|k|v kernel reduces them, records the token and gathers
// its embedding row. Step i feeds clip b at position h->d_pos[b] + i - 1.
// sampled: the sampler writes tk[:, i] from the full logits, and the next step gathers from tk (fused into
// layer 0 for 1..4 clips, the embedding kernel otherwise).
int decode_steps(vcl_handle* h, int32_t* tk, int B, int n_new, cudaStream_t st, int sampled) {
  const bool hand_off = B <= 4 && h->cfg.llm_layers > 0 && !sampled;
  for (int i = 1; i < n_new; ++i) {
    StepIo io;
    io.pos_dev = h->d_pos;
    io.sampled = sampled;
    if (hand_off && i > 1) {
      io.tok_from_partials = true; io.tok_store = tk + (i - 1); io.store_stride = n_new;
    } else {
      io.tok_in = tk + (i - 1); io.in_stride = n_new;
    }
    if (hand_off && i + 1 < n_new) io.partials_out = true;
    else { io.tok_out = tk + i; io.out_stride = n_new; }
    VCL_TRY(llm_decode_step(h, io, B, i - 1, st));
  }
  return 0;
}

// decode_steps from one captured graph per (B, n_new, sampled), sampled as h->sampler gives it. The positions (h->d_pos, written by the caller),
// the pad counts (h->d_npad) and the sampling table are read on the device, so new positions, padding or sampling
// settings replay the same graph. Bounded LRU cache (an entry holds thousands of nodes). A stream that cannot be
// captured runs the steps eagerly.
int run_decode_steps(vcl_handle* h, int32_t* tk, int B, int n_new, cudaStream_t st, int sampled) {
  GraphEntry* ge = nullptr;
  for (auto& g : h->graphs)
    if (g.B == B && g.n_new == n_new && g.sampled == sampled) ge = &g;
  const bool can_capture = (st != nullptr) && (st != cudaStreamLegacy);
  if (ge == nullptr && can_capture) {
    if (h->graphs.size() >= MAX_DECODE_GRAPHS) {
      size_t victim = 0;
      for (size_t i = 1; i < h->graphs.size(); ++i)
        if (h->graphs[i].last_use < h->graphs[victim].last_use) victim = i;
      cudaGraphExecDestroy(h->graphs[victim].exec);
      h->graphs.erase(h->graphs.begin() + victim);
    }
    const long long before = launch_count();
    VCL_CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const int rc = decode_steps(h, tk, B, n_new, st, sampled);
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamEndCapture(st, &graph);
    const long long nodes = launch_count() - before;
    count_launches(-nodes);  // captured, not executed
    if (rc != 0) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    if (e != cudaSuccess) {
      set_last_error("decode graph capture failed: %s", cudaGetErrorString(e));
      return -2;
    }
    cudaGraphExec_t exec = nullptr;
    e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) {
      set_last_error("decode graph instantiate failed: %s", cudaGetErrorString(e));
      return -2;
    }
    h->graphs.push_back({B, n_new, sampled, exec, nodes, 0});
    ge = &h->graphs.back();
  }
  if (ge == nullptr) return decode_steps(h, tk, B, n_new, st, sampled);
  ge->last_use = ++h->graph_clock;
  VCL_CUDA_OK(cudaGraphLaunch(ge->exec, st));
  count_launches(ge->kernels);
  return 0;
}

// The loop of vcl_llm_decode_loop and vcl_llm_slot_decode, with h->d_pos written by the caller: first_tok
// [B] is fed, n_new - 1 steps follow, and [B, n_new] tokens (first_tok included) go to out_tokens. The arg-max
// kernels unless one of the entries 0 .. B-1 of the sampling table samples or wants log-probs.
int decode_loop(vcl_handle* h, const int32_t* first_tok, int B, int n_new, int32_t* out_tokens, cudaStream_t st) {
  int32_t* tk = h->tokens;  // [B, n_new] row-major scratch
  if (first_tok != tk)
    VCL_CUDA_OK(cudaMemcpy2DAsync(tk, (size_t)n_new * sizeof(int32_t), first_tok, sizeof(int32_t),
                                  sizeof(int32_t), B, cudaMemcpyDeviceToDevice, st));
  if (n_new > 1) VCL_TRY(run_decode_steps(h, tk, B, n_new, st, h->sampler(0, B)));
  VCL_CUDA_OK(cudaMemcpyAsync(out_tokens, tk, (size_t)B * n_new * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  return 0;
}

}  // namespace

extern "C" {

int vcl_clip_encode(vcl_handle* h, const void* pixels, int pixel_format, int n_frames, int frame_h, int frame_w,
                    int n_layers, void* hidden_out, void* stream) {
  VCL_REQUIRE(h && pixels && hidden_out, "vcl_clip_encode: null argument");
  VCL_REQUIRE(frame_h == h->cfg.image_size && frame_w == h->cfg.image_size,
              "vcl_clip_encode: frames are %dx%d but the tower takes %dx%d (resize / crop them first)", frame_h,
              frame_w, h->cfg.image_size, h->cfg.image_size);
  cudaStream_t st = as_stream(stream);
  VCL_TRY(clip_forward(h, pixels, pixel_format, n_frames, n_layers, st));
  const size_t bytes = (size_t)n_frames * (h->P + 1) * h->cfg.clip_hidden * 2;
  VCL_CUDA_OK(cudaMemcpyAsync(hidden_out, h->v_h, bytes, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int vcl_st_pool(const void* feats, int in_dtype, int64_t frame_stride, int64_t patch_stride, int T,
                int P, int C, int n_temporal, void* out, int out_dtype, void* stream) {
  VCL_REQUIRE(feats && out, "vcl_st_pool: null argument");
  if (check_device() != 0) return -2;
  return launch_st_pool(feats, in_dtype, frame_stride, patch_stride, T, P, C, n_temporal, out, out_dtype,
                        as_stream(stream));
}

int vcl_clip_features(vcl_handle* h, const void* pixels, int pixel_format, int n_frames, int frame_h, int frame_w,
                      void* out, int out_dtype, void* stream) {
  VCL_REQUIRE(h && pixels && out, "vcl_clip_features: null argument");
  VCL_REQUIRE(frame_h == h->cfg.image_size && frame_w == h->cfg.image_size,
              "vcl_clip_features: frames are %dx%d but the tower takes %dx%d (resize / crop them first)", frame_h,
              frame_w, h->cfg.image_size, h->cfg.image_size);
  cudaStream_t st = as_stream(stream);
  VCL_REQUIRE(n_frames <= h->cfg.n_temporal, "vcl_clip_features: %d frames exceed the %d temporal slots",
              n_frames, h->cfg.n_temporal);
  VCL_TRY(clip_forward(h, pixels, pixel_format, n_frames, h->cfg.clip_layers, st));
  const int C = h->cfg.clip_hidden;
  // drop the CLS row by starting at row 1 of every frame
  return launch_st_pool(h->v_h + C, VCL_DTYPE_BF16, (long long)(h->P + 1) * C, C, n_frames, h->P, C,
                        h->cfg.n_temporal, out, out_dtype, st);
}

int vcl_llm_prefill(vcl_handle* h, const int64_t* ids, const void* video_feats,
                    const int32_t* vid_start, int B, int S, int n_layers, void* hidden_out,
                    float* logits_out, int32_t* next_tok, void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_prefill: null handle");
  VCL_NOT_PAGED(h, "vcl_llm_prefill");
  return llm_prefill(h, ids, video_feats, vid_start, B, S, n_layers, hidden_out, logits_out, next_tok, 1,
                     as_stream(stream));
}

int vcl_llm_prefill_states(vcl_handle* h, const int64_t* ids, const void* video_feats,
                           const int32_t* vid_start, int B, int S, void* states_out, float* logits_out,
                           void* stream) {
  VCL_REQUIRE(h != nullptr && states_out != nullptr, "vcl_llm_prefill_states: null argument");
  VCL_NOT_PAGED(h, "vcl_llm_prefill_states");
  return llm_prefill(h, ids, video_feats, vid_start, B, S, h->cfg.llm_layers, nullptr, logits_out, nullptr, 1,
                     as_stream(stream), 0, states_out);
}

int vcl_llm_prefill_append(vcl_handle* h, const int64_t* ids, int B, int S, int start_pos, void* hidden_out,
                           float* logits_out, int32_t* next_tok, void* stream) {
  VCL_REQUIRE(h != nullptr && ids != nullptr, "vcl_llm_prefill_append: null argument");
  VCL_NOT_PAGED(h, "vcl_llm_prefill_append");
  VCL_REQUIRE(start_pos > 0, "vcl_llm_prefill_append: start_pos must be > 0 (use vcl_llm_prefill for a new sequence)");
  return llm_prefill(h, ids, nullptr, nullptr, B, S, h->cfg.llm_layers, hidden_out, logits_out, next_tok, 1,
                     as_stream(stream), start_pos);
}

int vcl_llm_decode_step(vcl_handle* h, const int32_t* tok_in, int B, int pos, float* logits_out,
                        int32_t* tok_out, void* stream) {
  VCL_REQUIRE(h && tok_in, "vcl_llm_decode_step: null argument");
  VCL_NOT_PAGED(h, "vcl_llm_decode_step");
  VCL_REQUIRE(h->llm_loaded, "LLM weights are not loaded");
  VCL_REQUIRE(B > 0 && B <= h->cfg.max_batch, "B=%d outside 1..%d", B, h->cfg.max_batch);
  StepIo io;
  io.tok_in = tok_in; io.logits_out = logits_out; io.tok_out = tok_out; io.sampled = h->sampler(0, B);
  return llm_decode_step(h, io, B, pos, as_stream(stream));
}

int vcl_llm_decode_loop(vcl_handle* h, const int32_t* first_tok, int B, int S, int n_new,
                        int32_t* out_tokens, void* stream) {
  VCL_REQUIRE(h && first_tok && out_tokens, "vcl_llm_decode_loop: null argument");
  VCL_NOT_PAGED(h, "vcl_llm_decode_loop");
  VCL_REQUIRE(h->llm_loaded, "LLM weights are not loaded");
  VCL_REQUIRE(B > 0 && B <= h->cfg.max_batch, "B=%d outside 1..%d", B, h->cfg.max_batch);
  VCL_REQUIRE(n_new >= 1 && S + n_new <= h->cfg.max_seq + 1, "S + n_new = %d exceeds max_seq %d", S + n_new,
              h->cfg.max_seq);
  VCL_REQUIRE(S >= h->npad_max, "S = %d lies inside the left padding (%d columns)", S, h->npad_max);
  cudaStream_t st = as_stream(stream);
  if (n_new > 1) VCL_TRY(launch_fill_int(h->d_pos, S, B, st));
  return decode_loop(h, first_tok, B, n_new, out_tokens, st);
}

int vcl_llm_slot_prefill(vcl_handle* h, int slot, const int64_t* ids, const void* video_feats,
                         const int32_t* vid_start, int S, int32_t* next_tok, void* stream) {
  VCL_REQUIRE(h && ids && vid_start && next_tok, "vcl_llm_slot_prefill: null argument");
  VCL_REQUIRE(h->llm_loaded, "LLM weights are not loaded");
  VCL_REQUIRE(slot >= 0 && slot < h->n_slots_max(), "vcl_llm_slot_prefill: slot %d outside 0..%d (%s)", slot,
              h->n_slots_max() - 1, h->slots_note().c_str());
  // a paged cache: the packed prefill of one prompt, bit for bit the same (vcl_llm_slots_prefill)
  if (h->paged()) return vcl_llm_slots_prefill(h, 1, &slot, &S, ids, video_feats, vid_start, next_tok, stream);
  return llm_prefill(h, ids, video_feats, vid_start, 1, S, h->cfg.llm_layers, nullptr, nullptr, next_tok, 1,
                     as_stream(stream), 0, nullptr, nullptr, slot);
}

// The packed prefill of n checked sequences (kernels.h): sequence i is rows start_i .. start_i + len_i - 1 of its
// prompt (start_host null: 0) into slot slots_host[i]; flash_host[i] (null: none) puts it on the flash attention
// kernel. One host-to-device copy of the map, then the layer stack.
static int packed_prefill(vcl_handle* h, int n, const int32_t* slots_host, const int32_t* start_host,
                   const int32_t* len_host, const int* flash_host, long long M, int S_max, const int64_t* ids,
                   const void* video_feats, const int32_t* vid_start, int32_t* next_tok, cudaStream_t st) {
  std::vector<int> map(pack_elems(M), 0);
  int* p = map.data();
  int pack_attn = 0;
  for (int i = 0, r = 0; i < n; ++i) {
    const int start = start_host ? start_host[i] : 0, len = len_host[i];
    const bool fl = flash_host != nullptr && flash_host[i];
    pack_attn |= fl ? 2 : 1;
    pack_off(p)[i] = r; pack_len(p)[i] = fl ? 0 : len; pack_slot(p)[i] = slots_host[i];
    pack_last(p)[i] = r + len - 1; pack_start(p)[i] = start; pack_end(p)[i] = start + len;
    for (int j = 0; j < len; ++j, ++r) {
      pack_row(p, r)[0] = i; pack_row(p, r)[1] = start + j;
    }
  }
  VCL_CUDA_OK(cudaMemcpyAsync(h->d_pack, p, map.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  int sampled = 0;
  for (int i = 0; i < n; ++i) sampled = std::max(sampled, h->sampler(slots_host[i], 1));
  return llm_prefill(h, ids, video_feats, vid_start, n, S_max, h->cfg.llm_layers, nullptr, nullptr, next_tok, 1, st,
                     0, nullptr, nullptr, 0, (int)M, sampled, pack_attn);
}

int vcl_llm_slots_prefill(vcl_handle* h, int n, const int32_t* slots_host, const int32_t* seq_len_host,
                          const int64_t* ids, const void* video_feats, const int32_t* vid_start, int32_t* next_tok,
                          void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_slots_prefill: null handle");
  const vcl_config& c = h->cfg;
  VCL_REQUIRE(n >= 1 && n <= h->n_slots_max(), "vcl_llm_slots_prefill: n=%d outside 1..%d (%s)", n, h->n_slots_max(),
              h->slots_note().c_str());
  VCL_REQUIRE(slots_host && seq_len_host && ids && vid_start && next_tok, "vcl_llm_slots_prefill: null argument");
  VCL_REQUIRE(h->llm_loaded, "LLM weights are not loaded");
  const int s_lim = c.max_seq < 512 ? c.max_seq : 512;   // 512: the key limit of the wgmma prefill attention
  long long M = 0;
  int S_max = 0;
  for (int i = 0; i < n; ++i) {
    const int s = slots_host[i], len = seq_len_host[i];
    VCL_REQUIRE(s >= 0 && s < h->n_slots_max(), "vcl_llm_slots_prefill: slot %d outside 0..%d", s, h->n_slots_max() - 1);
    for (int j = 0; j < i; ++j)
      VCL_REQUIRE(slots_host[j] != s, "vcl_llm_slots_prefill: slot %d is given twice", s);
    VCL_REQUIRE(len >= 1 && len <= s_lim, "vcl_llm_slots_prefill: sequence %d has %d tokens, outside 1..%d", i, len,
                s_lim);
    M += len;
    S_max = len > S_max ? len : S_max;
  }
  // n <= max_batch sequences of at most min(512, max_seq) tokens: M fits the activations (max_batch * act_seq() rows)
  return packed_prefill(h, n, slots_host, nullptr, seq_len_host, nullptr, M, S_max, ids, video_feats, vid_start,
                        next_tok, as_stream(stream));
}

int vcl_llm_slots_prefill_chunk(vcl_handle* h, int n, const int32_t* slots_host, const int32_t* start_host,
                                const int32_t* len_host, const int32_t* total_host, const int64_t* ids,
                                const void* video_feats, const int32_t* vid_start, int32_t* next_tok, void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_slots_prefill_chunk: null handle");
  const vcl_config& c = h->cfg;
  VCL_REQUIRE(h->paged(), "vcl_llm_slots_prefill_chunk: the handle has a contiguous KV cache (kv_blocks 0), which "
              "prefills long prompts in one pass (vcl_llm_slot_prefill)");
  VCL_REQUIRE(n >= 1 && n <= h->n_slots_max(), "vcl_llm_slots_prefill_chunk: n=%d outside 1..%d (%s)", n,
              h->n_slots_max(), h->slots_note().c_str());
  VCL_REQUIRE(slots_host && start_host && len_host && total_host && ids && vid_start && next_tok,
              "vcl_llm_slots_prefill_chunk: null argument");
  VCL_REQUIRE(h->llm_loaded, "LLM weights are not loaded");
  long long M = 0;
  int S_max = 0;
  for (int i = 0; i < n; ++i) {
    const int s = slots_host[i], st0 = start_host[i], len = len_host[i], tot = total_host[i];
    VCL_REQUIRE(s >= 0 && s < h->n_slots_max(), "vcl_llm_slots_prefill_chunk: slot %d outside 0..%d", s,
                h->n_slots_max() - 1);
    for (int j = 0; j < i; ++j)
      VCL_REQUIRE(slots_host[j] != s, "vcl_llm_slots_prefill_chunk: slot %d is given twice", s);
    VCL_REQUIRE(st0 >= 0 && st0 % 64 == 0, "vcl_llm_slots_prefill_chunk: sequence %d starts at %d, not a multiple of "
                "64 (the query tiles of a chunk must be those of the whole prompt)", i, st0);
    VCL_REQUIRE(len >= 1 && len <= 512, "vcl_llm_slots_prefill_chunk: sequence %d has %d rows, outside 1..512", i, len);
    VCL_REQUIRE(st0 + len <= tot, "vcl_llm_slots_prefill_chunk: sequence %d: rows %d..%d past its prompt of %d tokens",
                i, st0, st0 + len - 1, tot);
    VCL_REQUIRE(tot <= c.max_seq, "vcl_llm_slots_prefill_chunk: sequence %d: prompt of %d tokens exceeds max_seq %d",
                i, tot, c.max_seq);
    VCL_REQUIRE(tot > 512 || (st0 == 0 && len == tot), "vcl_llm_slots_prefill_chunk: sequence %d: a prompt of %d <= "
                "512 tokens is prefilled whole (start 0, length %d), as vcl_llm_slots_prefill does", i, tot, tot);
    M += len;
    S_max = len > S_max ? len : S_max;
  }
  VCL_REQUIRE(M <= (long long)c.max_batch * h->act_seq(), "vcl_llm_slots_prefill_chunk: %lld rows exceed the "
              "activations (max_batch %d * %d)", M, c.max_batch, h->act_seq());
  std::vector<int> flash(n);
  for (int i = 0; i < n; ++i) flash[i] = total_host[i] > 512;
  return packed_prefill(h, n, slots_host, start_host, len_host, flash.data(), M, S_max, ids, video_feats, vid_start,
                        next_tok, as_stream(stream));
}

int vcl_llm_slots_prefill_append(vcl_handle* h, int n, const int32_t* slots_host, const int32_t* start_host,
                                 const int32_t* len_host, const int64_t* ids, int32_t* next_tok, void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_slots_prefill_append: null handle");
  const vcl_config& c = h->cfg;
  VCL_REQUIRE(h->paged(), "vcl_llm_slots_prefill_append: the handle has a contiguous KV cache (kv_blocks 0), which "
              "continues a sequence with vcl_llm_prefill_append");
  VCL_REQUIRE(n >= 1 && n <= h->n_slots_max(), "vcl_llm_slots_prefill_append: n=%d outside 1..%d (%s)", n,
              h->n_slots_max(), h->slots_note().c_str());
  VCL_REQUIRE(slots_host && start_host && len_host && ids && next_tok, "vcl_llm_slots_prefill_append: null argument");
  VCL_REQUIRE(h->llm_loaded, "LLM weights are not loaded");
  long long M = 0;
  int S_max = 0;
  for (int i = 0; i < n; ++i) {
    const int s = slots_host[i], st0 = start_host[i], len = len_host[i];
    VCL_REQUIRE(s >= 0 && s < h->n_slots_max(), "vcl_llm_slots_prefill_append: slot %d outside 0..%d", s,
                h->n_slots_max() - 1);
    for (int j = 0; j < i; ++j)
      VCL_REQUIRE(slots_host[j] != s, "vcl_llm_slots_prefill_append: slot %d is given twice", s);
    VCL_REQUIRE(st0 >= 1, "vcl_llm_slots_prefill_append: sequence %d starts at %d; a tail continues a cached "
                "sequence (start >= 1; vcl_llm_slots_prefill takes new prompts)", i, st0);
    VCL_REQUIRE(len >= 1 && len <= 512, "vcl_llm_slots_prefill_append: sequence %d has %d rows, outside 1..512", i, len);
    VCL_REQUIRE(st0 + len <= c.max_seq, "vcl_llm_slots_prefill_append: sequence %d: rows %d..%d outside the cache "
                "(max_seq %d)", i, st0, st0 + len - 1, c.max_seq);
    M += len;
    S_max = len > S_max ? len : S_max;
  }
  VCL_REQUIRE(M <= (long long)c.max_batch * h->act_seq(), "vcl_llm_slots_prefill_append: %lld rows exceed the "
              "activations (max_batch %d * %d)", M, c.max_batch, h->act_seq());
  // the kernel of the contiguous continued prefill (attention_prefill_tc_supported): wgmma up to 512 keys
  std::vector<int> flash(n);
  for (int i = 0; i < n; ++i) flash[i] = start_host[i] + len_host[i] > 512;
  return packed_prefill(h, n, slots_host, start_host, len_host, flash.data(), M, S_max, ids, nullptr, nullptr,
                        next_tok, as_stream(stream));
}

int vcl_llm_slot_decode(vcl_handle* h, const int32_t* first_tok, const int32_t* pos_host, int n_slots, int n_new,
                        int32_t* out_tokens, void* stream) {
  VCL_REQUIRE(h && first_tok && pos_host && out_tokens, "vcl_llm_slot_decode: null argument");
  VCL_REQUIRE(h->llm_loaded, "LLM weights are not loaded");
  VCL_REQUIRE(n_slots >= 1 && n_slots <= h->n_slots_max(), "vcl_llm_slot_decode: n_slots=%d outside 1..%d (%s)",
              n_slots, h->n_slots_max(), h->slots_note().c_str());
  VCL_REQUIRE(!h->padded, "vcl_llm_slot_decode: the cache is left-padded; slots are unpadded (start each one with "
              "vcl_llm_slot_prefill)");
  VCL_REQUIRE(n_new >= 1 && n_new <= h->cfg.max_seq, "vcl_llm_slot_decode: n_new=%d outside 1..max_seq %d", n_new,
              h->cfg.max_seq);
  for (int b = 0; b < n_slots; ++b)
    VCL_REQUIRE(pos_host[b] >= 0 && pos_host[b] + n_new - 1 <= h->cfg.max_seq,
                "vcl_llm_slot_decode: slot %d: pos %d + n_new - 1 = %d exceeds max_seq %d", b, pos_host[b],
                pos_host[b] + n_new - 1, h->cfg.max_seq);
  cudaStream_t st = as_stream(stream);
  if (n_new > 1)
    VCL_CUDA_OK(cudaMemcpyAsync(h->d_pos, pos_host, (size_t)n_slots * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  return decode_loop(h, first_tok, n_slots, n_new, out_tokens, st);
}

int vcl_llm_set_sampling(vcl_handle* h, int n, const int32_t* clips_host, const float* temperature_host,
                         const int32_t* top_k_host, const uint64_t* seed_host, void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_set_sampling: null handle");
  const int mb = h->cfg.max_batch;
  VCL_REQUIRE(n >= 1 && n <= mb, "vcl_llm_set_sampling: n=%d outside 1..%d", n, mb);
  VCL_REQUIRE(clips_host && temperature_host && top_k_host && seed_host, "vcl_llm_set_sampling: null argument");
  for (int i = 0; i < n; ++i) {
    const int b = clips_host[i];
    const float T = temperature_host[i];
    VCL_REQUIRE(b >= 0 && b < mb, "vcl_llm_set_sampling: clip %d outside 0..%d", b, mb - 1);
    for (int j = 0; j < i; ++j)
      VCL_REQUIRE(clips_host[j] != b, "vcl_llm_set_sampling: clip %d is given twice", b);
    VCL_REQUIRE(isfinite(T) && T >= 0.f, "vcl_llm_set_sampling: temperature %g of clip %d is not a finite value >= 0",
                (double)T, b);
    VCL_REQUIRE(top_k_host[i] >= 0, "vcl_llm_set_sampling: top_k %d of clip %d is negative", top_k_host[i], b);
  }
  unsigned char* hb = h->samp_host.data();
  for (int i = 0; i < n; ++i) {
    const int b = clips_host[i];
    h->samp_seed(hb)[b] = seed_host[i];
    h->samp_temp(hb)[b] = temperature_host[i];
    h->samp_topk(hb)[b] = top_k_host[i];
    h->samp_topp(hb)[b] = 1.f;
    h->samp_rep(hb)[b] = 1.f;
  }
  VCL_CUDA_OK(cudaMemcpyAsync(h->samp, hb, h->samp_host.size(), cudaMemcpyHostToDevice, as_stream(stream)));
  return 0;
}

// the token-set bitmap, all sets empty; the 32-bit sampler graphs captured without it are captured again
static int ensure_token_sets(vcl_handle* h, cudaStream_t st) {
  if (h->tset != nullptr) return 0;
  const size_t words = (size_t)h->cfg.max_batch * h->tset_words();
  VCL_TRY(dalloc(h, &h->tset, words));
  VCL_CUDA_OK(cudaMemsetAsync(h->tset, 0, words * 4, st));
  for (size_t i = h->graphs.size(); i-- > 0;)
    if (h->graphs[i].sampled == 2) {
      cudaGraphExecDestroy(h->graphs[i].exec);
      h->graphs.erase(h->graphs.begin() + i);
    }
  return 0;
}

int vcl_llm_set_sampling_ex(vcl_handle* h, int n, const int32_t* clips_host, const float* temperature_host,
                            const int32_t* top_k_host, const uint64_t* seed_host, const float* top_p_host,
                            const float* repetition_penalty_host, void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_set_sampling_ex: null handle");
  const int mb = h->cfg.max_batch;
  VCL_REQUIRE(n >= 1 && n <= mb, "vcl_llm_set_sampling_ex: n=%d outside 1..%d", n, mb);
  VCL_REQUIRE(clips_host && temperature_host && top_k_host && seed_host && top_p_host && repetition_penalty_host,
              "vcl_llm_set_sampling_ex: null argument");
  bool penalty = false;
  for (int i = 0; i < n; ++i) {
    const int b = clips_host[i];
    const float T = temperature_host[i], p = top_p_host[i], r = repetition_penalty_host[i];
    VCL_REQUIRE(b >= 0 && b < mb, "vcl_llm_set_sampling_ex: clip %d outside 0..%d", b, mb - 1);
    for (int j = 0; j < i; ++j)
      VCL_REQUIRE(clips_host[j] != b, "vcl_llm_set_sampling_ex: clip %d is given twice", b);
    VCL_REQUIRE(isfinite(T) && T >= 0.f, "vcl_llm_set_sampling_ex: temperature %g of clip %d is not a finite value "
                ">= 0", (double)T, b);
    VCL_REQUIRE(top_k_host[i] >= 0, "vcl_llm_set_sampling_ex: top_k %d of clip %d is negative", top_k_host[i], b);
    VCL_REQUIRE(p >= 0.f && p <= 1.f, "vcl_llm_set_sampling_ex: top_p %g of clip %d outside [0, 1]", (double)p, b);
    VCL_REQUIRE(isfinite(r) && r > 0.f, "vcl_llm_set_sampling_ex: repetition_penalty %g of clip %d is not a finite "
                "value > 0", (double)r, b);
    VCL_REQUIRE((p == 1.f && r == 1.f) || h->cfg.vocab <= VCL_SAMPLE_WIDE_MAX_V,
                "vcl_llm_set_sampling_ex: clip %d: top_p and repetition_penalty take a vocabulary of at most %d "
                "tokens (the sampler's shared memory), this model has %d", b, VCL_SAMPLE_WIDE_MAX_V, h->cfg.vocab);
    penalty = penalty || r != 1.f;
  }
  cudaStream_t st = as_stream(stream);
  if (penalty) VCL_TRY(ensure_token_sets(h, st));
  unsigned char* hb = h->samp_host.data();
  for (int i = 0; i < n; ++i) {
    const int b = clips_host[i];
    h->samp_seed(hb)[b] = seed_host[i];
    h->samp_temp(hb)[b] = temperature_host[i];
    h->samp_topk(hb)[b] = top_k_host[i];
    h->samp_topp(hb)[b] = top_p_host[i];
    h->samp_rep(hb)[b] = repetition_penalty_host[i];
  }
  VCL_CUDA_OK(cudaMemcpyAsync(h->samp, hb, h->samp_host.size(), cudaMemcpyHostToDevice, st));
  return 0;
}

int vcl_llm_set_token_set(vcl_handle* h, int entry, const int64_t* ids, int n, void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_set_token_set: null handle");
  VCL_REQUIRE(entry >= 0 && entry < h->cfg.max_batch, "vcl_llm_set_token_set: entry %d outside 0..%d", entry,
              h->cfg.max_batch - 1);
  VCL_REQUIRE(n >= 0 && (n == 0 || ids != nullptr), "vcl_llm_set_token_set: n=%d with %s ids", n,
              ids ? "given" : "null");
  VCL_REQUIRE(h->cfg.vocab <= VCL_SAMPLE_WIDE_MAX_V, "vcl_llm_set_token_set: the repetition penalty takes a "
              "vocabulary of at most %d tokens, this model has %d", VCL_SAMPLE_WIDE_MAX_V, h->cfg.vocab);
  cudaStream_t st = as_stream(stream);
  VCL_TRY(ensure_token_sets(h, st));
  return launch_token_set(h->tset + (size_t)entry * h->tset_words(), h->tset_words(),
                          reinterpret_cast<const long long*>(ids), n, h->cfg.vocab, st);
}

int vcl_llm_read_token_set(vcl_handle* h, int entry, uint32_t* bits_out, void* stream) {
  VCL_REQUIRE(h && bits_out, "vcl_llm_read_token_set: null argument");
  VCL_REQUIRE(entry >= 0 && entry < h->cfg.max_batch, "vcl_llm_read_token_set: entry %d outside 0..%d", entry,
              h->cfg.max_batch - 1);
  VCL_REQUIRE(h->tset != nullptr, "vcl_llm_read_token_set: no token set was ever set for this handle "
              "(vcl_llm_set_token_set, or a repetition penalty in vcl_llm_set_sampling_ex)");
  VCL_CUDA_OK(cudaMemcpyAsync(bits_out, h->tset + (size_t)entry * h->tset_words(), (size_t)h->tset_words() * 4,
                              cudaMemcpyDefault, as_stream(stream)));
  return 0;
}

int vcl_llm_set_logprobs(vcl_handle* h, int n, const int32_t* clips_host, const int32_t* top_n_host, void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_set_logprobs: null handle");
  const int mb = h->cfg.max_batch;
  VCL_REQUIRE(n >= 1 && n <= mb, "vcl_llm_set_logprobs: n=%d outside 1..%d", n, mb);
  VCL_REQUIRE(clips_host && top_n_host, "vcl_llm_set_logprobs: null argument");
  bool on = false;
  for (int i = 0; i < n; ++i) {
    const int b = clips_host[i], k = top_n_host[i];
    VCL_REQUIRE(b >= 0 && b < mb, "vcl_llm_set_logprobs: clip %d outside 0..%d", b, mb - 1);
    for (int j = 0; j < i; ++j)
      VCL_REQUIRE(clips_host[j] != b, "vcl_llm_set_logprobs: clip %d is given twice", b);
    VCL_REQUIRE(k >= -1 && k <= VCL_LOGPROBS_MAX, "vcl_llm_set_logprobs: top_n %d of clip %d outside -1..%d", k, b,
                VCL_LOGPROBS_MAX);
    on = on || k >= 0;
  }
  if (on && h->lp == nullptr) {
    VCL_TRY(dalloc(h, &h->lp, h->lp_plane() * 8));
    // the sampler graphs captured so far carry no log-prob buffer: capture them again
    for (size_t i = h->graphs.size(); i-- > 0;)
      if (h->graphs[i].sampled) {
        cudaGraphExecDestroy(h->graphs[i].exec);
        h->graphs.erase(h->graphs.begin() + i);
      }
  }
  unsigned char* hb = h->samp_host.data();
  for (int i = 0; i < n; ++i) h->samp_topn(hb)[clips_host[i]] = top_n_host[i];
  VCL_CUDA_OK(cudaMemcpyAsync(h->samp, hb, h->samp_host.size(), cudaMemcpyHostToDevice, as_stream(stream)));
  return 0;
}

int vcl_llm_read_logprobs(vcl_handle* h, int entry, int first_pos, int count, int32_t* ids_out, float* lp_out,
                          void* stream) {
  VCL_REQUIRE(h && ids_out && lp_out, "vcl_llm_read_logprobs: null argument");
  VCL_REQUIRE(h->lp != nullptr, "vcl_llm_read_logprobs: no log-probs were ever turned on for this handle "
              "(vcl_llm_set_logprobs)");
  VCL_REQUIRE(entry >= 0 && entry < h->cfg.max_batch, "vcl_llm_read_logprobs: entry %d outside 0..%d", entry,
              h->cfg.max_batch - 1);
  VCL_REQUIRE(first_pos >= 0 && count >= 1 && (long long)first_pos + count <= h->lp_rows(),
              "vcl_llm_read_logprobs: positions %d..%lld outside 0..%d", first_pos, (long long)first_pos + count - 1,
              h->lp_rows() - 1);
  constexpr int P = 1 + VCL_LOGPROBS_MAX;
  const size_t off = ((size_t)entry * h->lp_rows() + first_pos) * P, bytes = (size_t)count * P * 4;
  cudaStream_t st = as_stream(stream);
  VCL_CUDA_OK(cudaMemcpyAsync(ids_out, reinterpret_cast<const int*>(h->lp) + off, bytes, cudaMemcpyDefault, st));
  VCL_CUDA_OK(cudaMemcpyAsync(lp_out, reinterpret_cast<const float*>(h->lp) + h->lp_plane() + off, bytes,
                              cudaMemcpyDefault, st));
  return 0;
}

int vcl_llm_generate(vcl_handle* h, const int64_t* ids, const void* video_feats,
                     const int32_t* vid_start, int B, int S, int n_new, int32_t* out_tokens,
                     void* stream) {
  VCL_REQUIRE(h && out_tokens, "vcl_llm_generate: null argument");
  VCL_NOT_PAGED(h, "vcl_llm_generate");
  VCL_REQUIRE(n_new >= 1 && S + n_new <= h->cfg.max_seq + 1, "S + n_new = %d exceeds max_seq %d", S + n_new,
              h->cfg.max_seq);
  cudaStream_t st = as_stream(stream);
  VCL_TRY(llm_prefill(h, ids, video_feats, vid_start, B, S, h->cfg.llm_layers, nullptr, nullptr, h->tokens,
                      n_new, st));
  return vcl_llm_decode_loop(h, h->tokens, B, S, n_new, out_tokens, stream);
}

int vcl_llm_prefill_padded(vcl_handle* h, const int64_t* ids, const void* video_feats, const int32_t* vid_start,
                           const int32_t* n_pad_host, int B, int S, int n_layers, void* hidden_out,
                           float* logits_out, int32_t* next_tok, void* stream) {
  VCL_REQUIRE(h != nullptr && n_pad_host != nullptr, "vcl_llm_prefill_padded: null argument");
  VCL_NOT_PAGED(h, "vcl_llm_prefill_padded");
  return llm_prefill(h, ids, video_feats, vid_start, B, S, n_layers, hidden_out, logits_out, next_tok, 1,
                     as_stream(stream), 0, nullptr, n_pad_host);
}

int vcl_llm_generate_padded(vcl_handle* h, const int64_t* ids, const void* video_feats, const int32_t* vid_start,
                            const int32_t* n_pad_host, int B, int S, int n_new, int32_t* out_tokens, void* stream) {
  VCL_REQUIRE(h && out_tokens && n_pad_host, "vcl_llm_generate_padded: null argument");
  VCL_NOT_PAGED(h, "vcl_llm_generate_padded");
  VCL_REQUIRE(n_new >= 1 && S + n_new <= h->cfg.max_seq + 1, "S + n_new = %d exceeds max_seq %d", S + n_new,
              h->cfg.max_seq);
  cudaStream_t st = as_stream(stream);
  VCL_TRY(llm_prefill(h, ids, video_feats, vid_start, B, S, h->cfg.llm_layers, nullptr, nullptr, h->tokens,
                      n_new, st, 0, nullptr, n_pad_host));
  return vcl_llm_decode_loop(h, h->tokens, B, S, n_new, out_tokens, stream);
}

int vcl_llm_score(vcl_handle* h, const int64_t* ids, const void* video_feats, const int32_t* vid_start,
                  const int32_t* n_pad_host, int B, int S, const int64_t* labels, void* logits_out, float* nll_out,
                  float* loss_out, void* stream) {
  VCL_REQUIRE(h != nullptr, "vcl_llm_score: null handle");
  VCL_NOT_PAGED(h, "vcl_llm_score");
  VCL_REQUIRE(labels != nullptr || (nll_out == nullptr && loss_out == nullptr),
              "vcl_llm_score: nll_out / loss_out need labels");
  cudaStream_t st = as_stream(stream);
  VCL_TRY(llm_prefill(h, ids, video_feats, vid_start, B, S, h->cfg.llm_layers, nullptr, nullptr, nullptr, 1, st, 0,
                      nullptr, n_pad_host));
  if (logits_out == nullptr && labels == nullptr) return 0;
  return score_tail(h, B, S, labels, reinterpret_cast<bf16*>(logits_out), nll_out, loss_out, st);
}

long long vcl_launch_count(void) { return launch_count(); }

int vcl_kv_cache_copy(vcl_handle* h, int layer, int write, void* k, void* v, void* stream) {
  VCL_REQUIRE(h && k && v, "vcl_kv_cache_copy: null argument");
  VCL_REQUIRE(!h->paged(), "vcl_kv_cache_copy: this handle has a paged KV cache (kv_blocks %d): use vcl_kv_block_copy",
              h->cfg.kv_blocks);
  VCL_REQUIRE(layer >= 0 && layer < h->cfg.llm_layers, "vcl_kv_cache_copy: layer %d outside 0..%d", layer,
              h->cfg.llm_layers - 1);
  const size_t bytes = h->cache_layer_elems() * sizeof(bf16);
  cudaStream_t st = as_stream(stream);
  if (write) {
    VCL_CUDA_OK(cudaMemcpyAsync(kc_layer(h, layer), k, bytes, cudaMemcpyDeviceToDevice, st));
    VCL_CUDA_OK(cudaMemcpyAsync(vc_layer(h, layer), v, bytes, cudaMemcpyDeviceToDevice, st));
  } else {
    VCL_CUDA_OK(cudaMemcpyAsync(k, kc_layer(h, layer), bytes, cudaMemcpyDeviceToDevice, st));
    VCL_CUDA_OK(cudaMemcpyAsync(v, vc_layer(h, layer), bytes, cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

int vcl_llm_set_block_table(vcl_handle* h, const int32_t* table_host, void* stream) {
  VCL_REQUIRE(h && table_host, "vcl_llm_set_block_table: null argument");
  VCL_REQUIRE(h->paged(), "vcl_llm_set_block_table: the handle has a contiguous KV cache (kv_blocks 0)");
  const int nb = h->cfg.kv_blocks, row = h->table_row();
  std::vector<int> owner(nb, -1);    // the first entry that names each block
  for (size_t i = 0; i < h->table_host.size(); ++i) {
    const int blk = table_host[i];
    VCL_REQUIRE(blk >= 0 && blk < nb, "vcl_llm_set_block_table: slot %d, block %d: entry %d outside 0..%d",
                (int)(i / row), (int)(i % row), blk, nb - 1);
    VCL_REQUIRE(blk == 0 || owner[blk] < 0,
                "vcl_llm_set_block_table: block %d appears twice (slot %d block %d and slot %d block %d); only the "
                "park block 0 may be shared", blk, blk ? owner[blk] / row : 0, blk ? owner[blk] % row : 0,
                (int)(i / row), (int)(i % row));
    if (blk != 0) owner[blk] = (int)i;
  }
  memcpy(h->table_host.data(), table_host, h->table_host.size() * sizeof(int));
  VCL_CUDA_OK(cudaMemcpyAsync(h->d_table, h->table_host.data(), h->table_host.size() * sizeof(int),
                              cudaMemcpyHostToDevice, as_stream(stream)));
  return 0;
}

int vcl_kv_block_copy(vcl_handle* h, int block, int write, void* buf, void* stream) {
  VCL_REQUIRE(h && buf, "vcl_kv_block_copy: null argument");
  VCL_REQUIRE(h->paged(), "vcl_kv_block_copy: the handle has a contiguous KV cache (kv_blocks 0)");
  VCL_REQUIRE(block >= 0 && block < h->cfg.kv_blocks, "vcl_kv_block_copy: block %d outside 0..%d", block,
              h->cfg.kv_blocks - 1);
  bf16* blk = h->pool + (size_t)block * h->block_elems();
  const size_t bytes = h->block_elems() * sizeof(bf16);
  cudaStream_t st = as_stream(stream);
  if (write) VCL_CUDA_OK(cudaMemcpyAsync(blk, buf, bytes, cudaMemcpyDefault, st));
  else VCL_CUDA_OK(cudaMemcpyAsync(buf, blk, bytes, cudaMemcpyDefault, st));
  return 0;
}

// ---- single-operator entry points ----
int vcl_op_gemm(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc,
                const void* bias, const void* residual, int64_t ldr, int M, int N, int K, int act,
                int block_n, void* stream) {
  return vcl_op_gemm_ex(A, lda, W, ldw, C, ldc, bias, residual, ldr, M, N, K, act, block_n, 0, stream);
}

int vcl_op_gemm_ex(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc,
                   const void* bias, const void* residual, int64_t ldr, int M, int N, int K, int act,
                   int block_n, int cluster, void* stream) {
  if (check_device() != 0) return -2;
  static bool inited = false;
  if (!inited) {
    VCL_TRY(init_gemm_kernels());
    inited = true;
  }
  return gemm(reinterpret_cast<const bf16*>(A), lda, reinterpret_cast<const bf16*>(W), ldw,
              reinterpret_cast<bf16*>(C), ldc, reinterpret_cast<const bf16*>(bias),
              reinterpret_cast<const bf16*>(residual), ldr, M, N, K, act, as_stream(stream), block_n, cluster);
}

int vcl_op_cross_entropy(const void* logits, int64_t ld, const int64_t* labels, int rows, int V, float* nll_out,
                         float* loss_out, void* stream) {
  if (check_device() != 0) return -2;
  VCL_REQUIRE(logits != nullptr && labels != nullptr && nll_out != nullptr,
              "vcl_op_cross_entropy: logits, labels and nll_out are required");
  const long long* lab = reinterpret_cast<const long long*>(labels);
  VCL_TRY(launch_cross_entropy(reinterpret_cast<const bf16*>(logits), ld, V, lab, 0, rows, 0, nll_out, nullptr,
                               as_stream(stream)));
  return loss_out != nullptr ? launch_nll_mean(nll_out, lab, rows, 0, nullptr, loss_out, as_stream(stream)) : 0;
}

}  // extern "C"

namespace {

// vcl_op_sample / vcl_op_sample_logprobs / vcl_op_sample_ex: top_n_host null, or log-prob rows
// [B][1 + VCL_LOGPROBS_MAX] to ids_out / lp_out; top_p_host null (the 16-bit sampler), or the 32-bit sampler with
// top_p_host, rep_host and the token sets tset [B][ceil(V / 32)] (device, may be null)
int op_sample(const char* name, const float* logits, int64_t ld, int B, int V, const float* temperature_host,
              const int32_t* top_k_host, const uint64_t* seed_host, const int32_t* counter_host,
              const int32_t* top_n_host, int32_t* tok_out, int32_t* ids_out, float* lp_out, void* stream,
              const float* top_p_host = nullptr, const float* rep_host = nullptr, uint32_t* tset = nullptr) {
  if (check_device() != 0) return -2;
  VCL_REQUIRE(logits && temperature_host && top_k_host && seed_host && counter_host && tok_out, "%s: null argument",
              name);
  VCL_REQUIRE(B >= 1, "%s: B=%d", name, B);
  const bool wide = top_p_host != nullptr;
  if (wide) {
    VCL_REQUIRE(rep_host != nullptr, "%s: null argument", name);
    VCL_REQUIRE(V >= 1 && V <= VCL_SAMPLE_WIDE_MAX_V, "%s: V=%d outside 1..%d (the 32-bit sampler's shared memory)",
                name, V, VCL_SAMPLE_WIDE_MAX_V);
    for (int b = 0; b < B; ++b)
      VCL_REQUIRE(top_p_host[b] >= 0.f && top_p_host[b] <= 1.f && isfinite(rep_host[b]) && rep_host[b] > 0.f,
                  "%s: row %d: top_p %g outside [0, 1] or repetition_penalty %g not a finite value > 0", name, b,
                  (double)top_p_host[b], (double)rep_host[b]);
  }
  for (int b = 0; b < B; ++b)
    VCL_REQUIRE(isfinite(temperature_host[b]) && temperature_host[b] >= 0.f && top_k_host[b] >= 0 &&
                counter_host[b] >= 0, "%s: row %d: temperature %g, top_k %d, counter %d", name, b,
                (double)temperature_host[b], top_k_host[b], counter_host[b]);
  if (top_n_host != nullptr)
    for (int b = 0; b < B; ++b)
      VCL_REQUIRE(top_n_host[b] >= -1 && top_n_host[b] <= VCL_LOGPROBS_MAX, "%s: row %d: top_n %d outside -1..%d",
                  name, b, top_n_host[b], VCL_LOGPROBS_MAX);
  // the per-row settings in one stream-ordered block: [B] seeds, temperatures, top_k, counters, top_n, top_p, penalties
  std::vector<unsigned char> hb((size_t)B * (wide ? 32 : 24));
  memcpy(hb.data(), seed_host, (size_t)B * 8);
  memcpy(hb.data() + (size_t)B * 8, temperature_host, (size_t)B * 4);
  memcpy(hb.data() + (size_t)B * 12, top_k_host, (size_t)B * 4);
  memcpy(hb.data() + (size_t)B * 16, counter_host, (size_t)B * 4);
  if (top_n_host != nullptr) memcpy(hb.data() + (size_t)B * 20, top_n_host, (size_t)B * 4);
  if (wide) {
    memcpy(hb.data() + (size_t)B * 24, top_p_host, (size_t)B * 4);
    memcpy(hb.data() + (size_t)B * 28, rep_host, (size_t)B * 4);
  }
  cudaStream_t st = as_stream(stream);
  unsigned char* d = nullptr;
  VCL_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&d), hb.size(), st));
  VCL_CUDA_OK(cudaMemcpyAsync(d, hb.data(), hb.size(), cudaMemcpyHostToDevice, st));
  SampleArgs sa;
  sa.logits = logits; sa.ld = ld; sa.V = V; sa.B = B;
  sa.seed = reinterpret_cast<const unsigned long long*>(d);
  sa.temperature = reinterpret_cast<const float*>(d + (size_t)B * 8);
  sa.top_k = reinterpret_cast<const int*>(d + (size_t)B * 12);
  sa.col_dev = reinterpret_cast<const int*>(d + (size_t)B * 16);
  sa.out = tok_out;
  if (top_n_host != nullptr) {   // row b's places at ids_out / lp_out + b * (1 + VCL_LOGPROBS_MAX), any counter
    sa.top_n = reinterpret_cast<const int*>(d + (size_t)B * 20);
    sa.lp_id = ids_out; sa.lp_val = lp_out; sa.lp_entry = 1 + VCL_LOGPROBS_MAX; sa.lp_pos = 0; sa.lp_rows = 0x7fffffff;
  }
  if (wide) {
    sa.top_p = reinterpret_cast<const float*>(d + (size_t)B * 24);
    sa.rep = reinterpret_cast<const float*>(d + (size_t)B * 28);
    sa.tset = tset; sa.tset_words = (V + 31) / 32;
  }
  const int rc = launch_sample(sa, st);
  VCL_CUDA_OK(cudaFreeAsync(d, st));
  return rc;
}

}  // namespace

extern "C" {

int vcl_op_sample(const float* logits, int64_t ld, int B, int V, const float* temperature_host,
                  const int32_t* top_k_host, const uint64_t* seed_host, const int32_t* counter_host, int32_t* tok_out,
                  void* stream) {
  return op_sample("vcl_op_sample", logits, ld, B, V, temperature_host, top_k_host, seed_host, counter_host, nullptr,
                   tok_out, nullptr, nullptr, stream);
}

int vcl_op_sample_logprobs(const float* logits, int64_t ld, int B, int V, const float* temperature_host,
                           const int32_t* top_k_host, const uint64_t* seed_host, const int32_t* counter_host,
                           const int32_t* top_n_host, int32_t* tok_out, int32_t* ids_out, float* lp_out,
                           void* stream) {
  VCL_REQUIRE(top_n_host && ids_out && lp_out, "vcl_op_sample_logprobs: null argument");
  return op_sample("vcl_op_sample_logprobs", logits, ld, B, V, temperature_host, top_k_host, seed_host, counter_host,
                   top_n_host, tok_out, ids_out, lp_out, stream);
}

int vcl_op_sample_ex(const float* logits, int64_t ld, int B, int V, const float* temperature_host,
                     const int32_t* top_k_host, const uint64_t* seed_host, const int32_t* counter_host,
                     const float* top_p_host, const float* repetition_penalty_host, uint32_t* token_sets,
                     const int32_t* top_n_host, int32_t* tok_out, int32_t* ids_out, float* lp_out, void* stream) {
  VCL_REQUIRE(top_p_host && repetition_penalty_host, "vcl_op_sample_ex: null argument");
  VCL_REQUIRE(top_n_host == nullptr || (ids_out && lp_out), "vcl_op_sample_ex: log-probs need ids_out and lp_out");
  return op_sample("vcl_op_sample_ex", logits, ld, B, V, temperature_host, top_k_host, seed_host, counter_host,
                   top_n_host, tok_out, ids_out, lp_out, stream, top_p_host, repetition_penalty_host, token_sets);
}

int vcl_op_layernorm(const void* x, void* y, const void* w, const void* b, int rows, int D, float eps,
                     void* stream) {
  if (check_device() != 0) return -2;
  return launch_layernorm(reinterpret_cast<const bf16*>(x), D, reinterpret_cast<bf16*>(y), D,
                          reinterpret_cast<const bf16*>(w), reinterpret_cast<const bf16*>(b), rows, D, eps,
                          as_stream(stream));
}

int vcl_op_rmsnorm(const void* x, void* y, const void* w, int rows, int D, float eps, void* stream) {
  if (check_device() != 0) return -2;
  return launch_rmsnorm(reinterpret_cast<const bf16*>(x), D, reinterpret_cast<bf16*>(y), D,
                        reinterpret_cast<const bf16*>(w), rows, D, eps, as_stream(stream));
}

int vcl_op_attention(const void* q, const void* k, const void* v, void* o, int B, int S, int H,
                     int head_dim, float scale, int causal, void* stream) {
  if (check_device() != 0) return -2;
  static bool inited = false;
  if (!inited) {
    VCL_TRY(init_attention_kernels());
    inited = true;
  }
  AttnArgs a;
  const long long sb = (long long)S * H * head_dim, sh = head_dim, ss = (long long)H * head_dim;
  a.q = reinterpret_cast<const bf16*>(q); a.q_sb = sb; a.q_sh = sh; a.q_ss = ss;
  a.k = reinterpret_cast<const bf16*>(k); a.k_sb = sb; a.k_sh = sh; a.k_ss = ss;
  a.v = reinterpret_cast<const bf16*>(v); a.v_sb = sb; a.v_sh = sh; a.v_ss = ss;
  a.o = reinterpret_cast<bf16*>(o); a.o_sb = sb; a.o_sh = sh; a.o_ss = ss;
  a.B = B; a.H = H; a.S = S; a.head_dim = head_dim; a.scale = scale; a.causal = causal;
  return launch_attention(a, as_stream(stream));
}

int vcl_op_attention_vit(const void* qkv, void* out, int n_frames, int S, int H, void* stream) {
  if (check_device() != 0) return -2;
  static bool inited = false;
  if (!inited) {
    VCL_TRY(init_attention_kernels());
    inited = true;
  }
  return launch_attention_vit(reinterpret_cast<const bf16*>(qkv), reinterpret_cast<bf16*>(out), n_frames, S, H,
                                 H * 64, as_stream(stream));
}

int vcl_op_gemv(const void* x, const void* W, void* out, const void* res, const void* norm_w,
                float eps, int B, int N, int K, void* stream) {
  if (check_device() != 0) return -2;
  VCL_REQUIRE(B >= 1 && B <= 64, "vcl_op_gemv: B=%d outside 1..64 (more rows take the GEMM)", B);
  VCL_REQUIRE(gemv_fits(B, N, K, norm_w != nullptr),
              "vcl_op_gemv: B=%d N=%d K=%d is outside the decode kernels' range", B, N, K);
  static bool inited = false;
  if (!inited) {
    VCL_TRY(init_gemv_kernels());
    inited = true;
  }
  GemvArgs g;
  g.x = reinterpret_cast<const bf16*>(x); g.ldx = K;
  g.B = B; g.N = N; g.K = K; g.norm_w = reinterpret_cast<const bf16*>(norm_w); g.eps = eps;
  // the decode kernels read the slot-ordered copy of the matrix. It is built here and kept for the next call
  // with the same matrix (this entry point is a test / micro-benchmark hook, not a hot path); the copy is only
  // REUSED when VCL_OP_GEMV_CACHE is set (tools/microbench.py), because a caller may hand in a different
  // matrix at a recycled address
  static const void* c_W = nullptr; static int c_N = 0, c_K = 0; static bf16* c_tiled = nullptr;
  if (c_W != W || c_N != N || c_K != K || getenv("VCL_OP_GEMV_CACHE") == nullptr) {
    cudaStreamSynchronize(as_stream(stream));
    if (c_tiled != nullptr) cudaFree(c_tiled);
    c_tiled = nullptr; c_W = nullptr;
    VCL_CUDA_OK(cudaMalloc(&c_tiled, gemv_tiled_elems(N, K) * sizeof(bf16)));
    const int rc0 = launch_gemv_repack(reinterpret_cast<const bf16*>(W), c_tiled, N, K, false, as_stream(stream));
    if (rc0 != 0) { cudaFree(c_tiled); c_tiled = nullptr; return rc0; }
    c_W = W; c_N = N; c_K = K;
  }
  g.W_tiled = c_tiled;
  return op_gemv_run(g, out, res, eps, as_stream(stream));
}

int vcl_op_quantize_fp8(const void* W, int N, int K, void* w_deq, void* codes, float* scales, void* stream) {
  if (check_device() != 0) return -2;
  VCL_REQUIRE(W && w_deq && codes && scales, "vcl_op_quantize_fp8: null argument");
  return launch_gemv_quantize_fp8(reinterpret_cast<const bf16*>(W), reinterpret_cast<bf16*>(w_deq),
                                  reinterpret_cast<uint8_t*>(codes), scales, N, K, false, nullptr, as_stream(stream));
}

int vcl_op_gemv_fp8(const void* x, const void* W, void* out, const void* res, const void* norm_w,
                    float eps, int B, int N, int K, void* stream) {
  if (check_device() != 0) return -2;
  VCL_REQUIRE(B >= 1 && B <= 64, "vcl_op_gemv_fp8: B=%d outside 1..64 (more rows take the GEMM)", B);
  VCL_REQUIRE(gemv_fits(B, N, K, norm_w != nullptr, true),
              "vcl_op_gemv_fp8: B=%d N=%d K=%d is outside the decode kernels' range", B, N, K);
  static bool inited = false;
  if (!inited) {
    VCL_TRY(init_gemv_kernels());
    inited = true;
  }
  // the load-time quantizer into stream-ordered scratch (W itself is left as it is), then the fp8 ring kernels
  cudaStream_t st = as_stream(stream);
  unsigned char* scratch = nullptr;
  const size_t deq = (size_t)N * K * sizeof(bf16), cb = (gemv_tiled_elems(N, K) + 255) / 256 * 256;
  VCL_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&scratch), deq + cb + (size_t)N * sizeof(float), st));
  GemvArgs g;
  g.x = reinterpret_cast<const bf16*>(x); g.ldx = K;
  g.B = B; g.N = N; g.K = K; g.norm_w = reinterpret_cast<const bf16*>(norm_w); g.eps = eps;
  g.W_fp8 = scratch + deq; g.w_scale = reinterpret_cast<float*>(scratch + deq + cb);
  int rc = launch_gemv_quantize_fp8(reinterpret_cast<const bf16*>(W), reinterpret_cast<bf16*>(scratch),
                                    scratch + deq, reinterpret_cast<float*>(scratch + deq + cb), N, K, false, nullptr, st);
  if (rc == 0) rc = op_gemv_run(g, out, res, eps, st);
  VCL_CUDA_OK(cudaFreeAsync(scratch, st));
  return rc;
}

}  // extern "C"

namespace {

// out = x . W^T (+ res) by the decode kernels, with g's weights; 5..64 rows through the xwin re-layout
int op_gemv_run(GemvArgs g, void* out, const void* res, float eps, cudaStream_t st) {
  const int B = g.B, N = g.N, K = g.K;
  GemvEpilogue e;
  e.mode = GEMV_RES; e.out = reinterpret_cast<bf16*>(out); e.ldo = N; e.res = reinterpret_cast<const bf16*>(res); e.ldr = N;
  if (B >= 5) {
    // 5..64 rows: the xwin ring kernels; their input is normalised and re-laid out (xwin) by a launch of its own,
    // as on the decode path
    static bf16* xn = nullptr; static size_t xn_elems = 0;
    if (xn_elems < xwin_elems(B, K)) {
      cudaStreamSynchronize(st);
      if (xn) cudaFree(xn);
      VCL_CUDA_OK(cudaMalloc(&xn, xwin_elems(B, K) * sizeof(bf16)));
      xn_elems = xwin_elems(B, K);
    }
    VCL_TRY(launch_xwin_norm(g.x, K, xn, g.norm_w, B, K, eps, st));
    g.x = xn; g.norm_w = nullptr;
  }
  return launch_gemv(g, e, st);
}

}  // namespace

extern "C" {

int vcl_op_decode_attention(const void* q, int64_t q_ld, const void* k, const void* v, void* o, int B, int H,
                            int s_max, int kv_len, const int32_t* pos_dev, const int32_t* n_pad, float scale,
                            int o_xwin, void* stream) {
  if (check_device() != 0) return -2;
  VCL_REQUIRE(q && k && v && o && n_pad, "vcl_op_decode_attention: q, k, v, o and n_pad are required");
  VCL_REQUIRE(B > 0 && H > 0 && q_ld >= (int64_t)H * 128 && q_ld % 8 == 0,
              "vcl_op_decode_attention: B=%d H=%d q_ld=%lld", B, H, (long long)q_ld);
  return launch_decode_attention(reinterpret_cast<const bf16*>(q), q_ld, reinterpret_cast<const bf16*>(k),
                                 reinterpret_cast<const bf16*>(v), reinterpret_cast<bf16*>(o), (long long)H * 128, B,
                                 H, 128, s_max, kv_len, scale, as_stream(stream), pos_dev, o_xwin != 0, n_pad);
}

}  // extern "C"

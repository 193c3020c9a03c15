/* vcl.h -- C ABI of libvcl.so, the H100-native (sm_90a) replacement for the device side of
 * PG-Video-LLaVA's video-conversation inference path.
 *
 * The reference (mbzuai-oryx/Video-LLaVA) has no FFI or operator registry: its boundary is a set
 * of Python call sites that hand tensors to PyTorch/HF modules. Each entry point below states the
 * reference call it replaces (file:line relative to the reference tree; "$TF" = the installed
 * HuggingFace transformers, where the arithmetic the reference delegates to lives).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; the caller owns all memory
 *     passed in; the library owns its packed weights, activations and KV cache (allocated by
 *     vcl_create / vcl_load_*), freed by vcl_destroy;
 *   - 16-bit tensors are bf16 unless a dtype code says otherwise (0 = fp16, 1 = bf16);
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*) and never synchronised,
 *     except vcl_load_* which return after the repack has completed;
 *   - return value 0 = ok, negative = error; vcl_last_error() gives the message of the last
 *     failure on the calling thread's process (one handle per process/GPU, not thread-safe);
 *   - there is no CPU fallback: on a machine without an sm_90 (H100) device every compute entry point
 *     fails with an error.
 */
#ifndef VCL_H_
#define VCL_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VCL_VERSION 1

#define VCL_DTYPE_F16 0
#define VCL_DTYPE_BF16 1

#define VCL_PIXELS_BF16_NCHW 0 /* [N,3,H,W] bf16, already CLIP-normalised (inference.py:86-89)   */
#define VCL_PIXELS_U8_NHWC 1   /* [N,H,W,3] uint8 raw frames; (x/255-mean)/std applied on device */

#define VCL_WEIGHTS_BF16 0     /* the checkpoint's bf16 weights, as loaded (the default)                      */
#define VCL_WEIGHTS_FP8_E4M3 1 /* the language model's streamed matrices as E4M3 codes with power-of-two row
                                  scales (vcl_load_llm_weights_ex)                                            */

#define VCL_PROJ_LINEAR 0     /* nn.Linear(1024, D)            video_chatgpt/model/video_chatgpt.py:51-53 */
#define VCL_PROJ_MLP2X_GELU 1 /* Linear-GELU-Linear            model/multimodal_projector/builder.py:39-46 */

typedef struct vcl_handle vcl_handle;

typedef struct vcl_config {
  /* vision tower: CLIP ViT ($TF/models/clip/modeling_clip.py:647-693) */
  int32_t clip_layers;   /* encoder layers to EXECUTE; the path consumes hidden_states[-2]
                            (inference.py:94), i.e. num_hidden_layers - 1 (23 for ViT-L/14)   */
  int32_t clip_hidden;   /* 1024 */
  int32_t clip_inter;    /* 4096 */
  int32_t clip_heads;    /* 16 (head_dim must be 64) */
  int32_t image_size;    /* 224 or 336 */
  int32_t patch_size;    /* 14 */
  float clip_ln_eps;     /* 1e-5 */
  /* language model: LLaMA/Vicuna ($TF/models/llama/modeling_llama.py:355-425) */
  int32_t llm_layers;    /* 32 (7B) / 40 (13B) */
  int32_t llm_hidden;    /* 4096 / 5120 (head_dim must be 128) */
  int32_t llm_inter;     /* 11008 / 13824; at most 14336 (the 1..4-clip decode kernel stages the
                            down_proj input in shared memory): vcl_create rejects larger values */
  int32_t llm_heads;     /* 32 / 40 (kv heads == heads) */
  int32_t vocab;         /* 32003 after the three video tokens are added (eval/model_utils.py:114-119) */
  float rms_eps;         /* 1e-5 */
  float rope_theta;      /* 10000 */
  int32_t proj_type;     /* VCL_PROJ_* */
  int32_t n_temporal;    /* 100: temporal token slots (inference.py:31) */
  /* capacities */
  int32_t max_frames;    /* frames per vcl_clip_encode call */
  int32_t max_batch;     /* clips per prefill / decode call */
  int32_t max_seq;       /* prompt + generated tokens per clip */
  int32_t max_slots;     /* in-flight cache slots (vcl_llm_slot_*): 0 = min(max_batch, 16); otherwise
                            1 .. min(max_batch, 64), anything else is rejected by vcl_create. A capacity
                            only: the decode kernel is chosen by the clip count of each call */
  int32_t kv_blocks;     /* 0: the contiguous KV cache, [layer][max_batch][head][max_seq][128] for K and for V.
                            > 0: a PAGED cache of kv_blocks blocks instead (vcl_llm_set_block_table); at least 2,
                            block 0 being the park block. A paged handle serves the slot entry points only */
} vcl_config;

/* A named tensor in the layout of the HF/reference state_dict (row-major, bf16, on the device).
 * Names are the state_dict keys listed in SURVEY.md section 8a ("weight-name contract"). */
typedef struct vcl_tensor {
  const char* name;
  const void* data;
  int32_t ndim;
  int64_t shape[4];
} vcl_tensor;

int vcl_version(void);
const char* vcl_last_error(void);

/* Replaces the module construction in video_chatgpt/eval/model_utils.py:104-105,134-136. */
int vcl_create(vcl_handle** out, const vcl_config* cfg);
void vcl_destroy(vcl_handle* h);

/* Replace CLIPVisionModel.from_pretrained / VideoChatGPTLlamaForCausalLM.from_pretrained +
 * load_state_dict (eval/model_utils.py:104,122-127,134): repack into the kernel layouts
 * (fused q|k|v, interleaved gate/up, K-padded patch-embed matrix). Unknown names are ignored
 * (e.g. vision_model.post_layernorm.*, unused by the path); a missing required name is an error.
 * vcl_load_llm_weights additionally builds a decode-only copy of the streamed matrices in the slot
 * order of the decode kernels (+1x the LLM weight bytes; +0.5x with vcl_load_llm_weights_ex's fp8 format). */
int vcl_load_clip_weights(vcl_handle* h, const vcl_tensor* tensors, int n);
int vcl_load_llm_weights(vcl_handle* h, const vcl_tensor* tensors, int n);

/* vcl_load_llm_weights with a weight format for the five streamed matrices of the language model (fused
 * q|k|v, o_proj, interleaved gate|up, down_proj, lm_head; the embedding table, the norms, the projector and the
 * CLIP tower stay bf16). VCL_WEIGHTS_BF16 is vcl_load_llm_weights. VCL_WEIGHTS_FP8_E4M3, per row r of each
 * matrix W (after the fusion / interleave above):
 *   a_r = max_k |W[r,k]|; e_r = the smallest integer with a_r <= 448 * 2^e_r (0 for an all-zero row);
 *   q[r,k] = E4M3(W[r,k] * 2^-e_r), round to nearest even, subnormals included (torch's .to(float8_e4m3fn));
 *   W~[r,k] = q[r,k] * 2^e_r, which is exactly a bf16 number.
 * The load writes W~ over the row-major matrix, so prefill, decode beyond 16 clips and vcl_llm_score compute
 * with W~, and keeps the codes (slot order of the decode kernels, one byte each) and 2^e_r per row instead of
 * the bf16 decode copy: the decode kernels read half the bytes, and the engine holds about half the LLM weight
 * bytes less. Every output is then bit for bit that of a VCL_WEIGHTS_BF16 engine loaded with W~. Rejected: an
 * unknown format (before any allocation), a non-finite weight, and a row whose 2^e_r is not a normal fp32
 * number or whose W~ is not exactly a finite bf16 (a row maximum below ~1e-36); the message names the
 * state-dict tensor and row. */
int vcl_load_llm_weights_ex(vcl_handle* h, const vcl_tensor* tensors, int n, int weight_format);

/* vision_tower(pixel_values, output_hidden_states=True).hidden_states[k]
 * (video_chatgpt/inference.py:93-94, scripts/save_spatio_temporal_clip_features.py:116-120).
 * Runs `n_layers` encoder layers (<= clip_layers; pass clip_layers for hidden_states[-2]; 0 gives
 * hidden_states[0], the post-pre_layrnorm embeddings). hidden_out is [n_frames, 1+P, C] bf16 with
 * the CLS row kept, as in HF; callers slice [:, 1:]. frame_h / frame_w are the height and width of
 * the frames behind `pixels`: they must equal image_size (the image processor of the reference
 * resizes and crops, inference.py:86; raw frames of another size are an error, never read out of bounds). */
int vcl_clip_encode(vcl_handle* h, const void* pixels, int pixel_format, int n_frames, int frame_h, int frame_w,
                    int n_layers, void* hidden_out, void* stream);

/* get_spatio_temporal_features_torch (video_chatgpt/inference.py:13-44) and its numpy twin
 * get_spatio_temporal_features (scripts/save_spatio_temporal_clip_features.py:46-57).
 * feats element (t,p,c) at feats + t*frame_stride + p*patch_stride + c (strides in elements), so a
 * [T,1+P,C] hidden state can be pooled in place by pointing at row 1. out is [n_temporal+P, C]. */
int vcl_st_pool(const void* feats, int in_dtype, int64_t frame_stride, int64_t patch_stride, int T,
                int P, int C, int n_temporal, void* out, int out_dtype, void* stream);

/* vcl_clip_encode(clip_layers) + CLS drop + vcl_st_pool in one call: the per-video body of
 * scripts/save_spatio_temporal_clip_features.py:105-123 and inference.py:93-95. */
int vcl_clip_features(vcl_handle* h, const void* pixels, int pixel_format, int n_frames, int frame_h, int frame_w,
                      void* out, int out_dtype, void* stream);

/* VideoChatGPTLlamaForCausalLM.forward on a full prompt (video_chatgpt/model/video_chatgpt.py:82-175,
 * 193-251): token embedding, mm_projector on video_feats [B, n_temporal+P, 1024], splice after
 * <vid_start> (vid_start[b] = index of the row after which the video rows go: the <vid_start> token, or
 * -1 when the patch tokens start the row without one; VCL_NO_VIDEO marks a text-only row), n_layers
 * decoder layers filling the KV cache at positions [0, S).
 *   hidden_out  optional [B,S,D] bf16: output of decoder layer n_layers (n_layers = 0: the spliced
 *               input embeddings), i.e. HF hidden_states[n_layers]
 *   logits_out  optional [B,vocab] fp32: lm_head(norm(h)) at the LAST position only, rounded to
 *               bf16 like the reference's logits tensor (requires n_layers == llm_layers)
 *   next_tok    optional [B] int32: arg-max of those logits (lowest index wins ties) */
int vcl_llm_prefill(vcl_handle* h, const int64_t* ids, const void* video_feats,
                    const int32_t* vid_start, int B, int S, int n_layers, void* hidden_out,
                    float* logits_out, int32_t* next_tok, void* stream);
#define VCL_NO_VIDEO (-2147483647 - 1)

/* vcl_llm_prefill for a batch of prompts of different lengths, left-padded to one length S (HF's
 * tokenizer with padding_side="left" and its attention_mask). n_pad_host [B] int32 in HOST memory: row b
 * starts with n_pad_host[b] pad ids (0 <= n_pad_host[b] < S, checked), its real tokens fill columns
 * n_pad_host[b] .. S-1. Every clip is computed as if it ran alone: cache column c holds the token at RoPE
 * position c - n_pad_host[b], and a real query attends keys n_pad_host[b] .. its own column only. The outputs
 * of pad rows (hidden_out) are finite but unspecified; logits / next token come from column S-1 as in
 * vcl_llm_prefill. vid_start[b] stays a column of the padded row, and the video span must lie inside the real
 * tokens. The pad ids are looked up like any other id, so they must be valid (< vocab).
 *
 * Padding state. The pad counts describe the KV cache, and the handle keeps them (in a device array of
 * max_batch entries): vcl_llm_prefill_padded / vcl_llm_generate_padded set them, vcl_llm_prefill,
 * vcl_llm_prefill_states and vcl_llm_generate clear them, and vcl_llm_prefill_append, vcl_llm_decode_step and
 * vcl_llm_decode_loop continue whatever padding the cache has. All-zero pad counts are no padding: the call is
 * then exactly vcl_llm_prefill. */
int vcl_llm_prefill_padded(vcl_handle* h, const int64_t* ids, const void* video_feats, const int32_t* vid_start,
                           const int32_t* n_pad_host, int B, int S, int n_layers, void* hidden_out,
                           float* logits_out, int32_t* next_tok, void* stream);

/* forward(..., output_hidden_states=True) (video_chatgpt/model/video_chatgpt.py:205-218): the same
 * full-depth prefill, keeping every hidden state: states_out is [llm_layers + 1][B][S][D] bf16, entry i
 * = the raw output of decoder layer i (entry 0: the spliced input embeddings). HF returns the LAST
 * entry after the final RMSNorm; the caller applies it (vcl_op_rmsnorm with model.norm.weight). */
int vcl_llm_prefill_states(vcl_handle* h, const int64_t* ids, const void* video_feats,
                           const int32_t* vid_start, int B, int S, void* states_out, float* logits_out,
                           void* stream);

/* Continue a cached sequence: S more token ids per clip (text only, no video span) take positions
 * [start_pos, start_pos + S) and attend to everything already in the KV cache. This is the building
 * block for multi-turn conversations about one video: the reference re-runs the vision tower and the
 * whole prompt on every turn (video_chatgpt/chat.py:137-154, inference.py:86-112); with the cache of
 * the previous turn only the new question is prefilled. Outputs as in vcl_llm_prefill (hidden_out
 * [B,S,D] of the new positions; logits / next token at the last new position). start_pos must be the
 * number of positions the cache of every clip already holds (> 0). A left-padded cache
 * (vcl_llm_prefill_padded) stays padded: the new tokens continue each clip's RoPE positions and do not attend
 * to its pad columns; start_pos must lie past the padding. */
int vcl_llm_prefill_append(vcl_handle* h, const int64_t* ids, int B, int S, int start_pos, void* hidden_out,
                           float* logits_out, int32_t* next_tok, void* stream);

/* One cached decoding step (the `input_ids.shape[1] == 1` branch, model/video_chatgpt.py:103,
 * 253-257): tok_in [B] int32 are fed at position `pos` (= tokens already in the cache).
 * logits_out / tok_out as above. Used for teacher-forced parity checks. After a padded prefill the step
 * continues the padding (RoPE position pos - n_pad[b], pad keys not read); pos must lie past the padding. */
int vcl_llm_decode_step(vcl_handle* h, const int32_t* tok_in, int B, int pos, float* logits_out,
                        int32_t* tok_out, void* stream);

/* model.generate(input_ids, video_spatio_temporal_features=..., do_sample=False,
 * max_new_tokens=n_new) with EOS ignored (video_chatgpt/inference.py:105-112; greedy is the
 * benchmark's setting, BASELINE.md section 5): prefill + (n_new-1) decode steps, tokens chained on
 * the device, the decode loop replayed from a CUDA graph. out_tokens is [B, n_new] int32 (new
 * tokens only; the Python shim prepends the prompt as HF does).
 * The graph is captured once per (B, n_new) on a non-default stream: the prompt length S reaches the
 * kernels through device memory, so any S replays it; at most 6 graphs are kept (least recently used
 * first out). With 1-4 clips no arg-max / embedding kernel runs between two steps (the logits kernel
 * leaves per-CTA partial arg-max, the next step's first q|k|v kernel reduces them and gathers the row). */
int vcl_llm_generate(vcl_handle* h, const int64_t* ids, const void* video_feats,
                     const int32_t* vid_start, int B, int S, int n_new, int32_t* out_tokens,
                     void* stream);

/* The decode half of vcl_llm_generate on its own (so a caller can time prefill and decode
 * separately): first_tok [B] int32 is the token produced by the prefill; runs n_new-1 cached steps
 * at positions S, S+1, ... and writes [B, n_new] (first_tok included) to out_tokens. It continues the
 * cache's left padding, if any; the graph cache is keyed by (B, n_new) alone, because the positions and the
 * pad counts are read from device memory: one graph serves every S and every padding. */
int vcl_llm_decode_loop(vcl_handle* h, const int32_t* first_tok, int B, int S, int n_new,
                        int32_t* out_tokens, void* stream);

/* vcl_llm_generate for a left-padded batch: vcl_llm_prefill_padded + vcl_llm_decode_loop (padding as
 * described at vcl_llm_prefill_padded; out_tokens [B, n_new] int32, new tokens only). */
int vcl_llm_generate_padded(vcl_handle* h, const int64_t* ids, const void* video_feats, const int32_t* vid_start,
                            const int32_t* n_pad_host, int B, int S, int n_new, int32_t* out_tokens, void* stream);

/* In-flight (continuous) batching: every clip of the KV cache is a SLOT that holds its own sequence at its own
 * length, so a finished request's slot takes the next queued request while the other slots keep decoding.
 * There are max_slots slots (vcl_config; 0 means min(max_batch, 16), at most min(max_batch, 64)). Slots are
 * unpadded. Decode projections by clip count: 1..4 gemv_tc, 5..64 gemv_tcw with 1 / 2 / 4 clip groups at 5..16 /
 * 17..32 / 33..64 clips (the ring kernels of decode_gemv.cu, each streaming every weight byte once per step), more
 * than 64 the prefill GEMM.
 *
 * vcl_llm_slot_prefill: vcl_llm_prefill of ONE prompt (ids [1,S], video_feats [1, n_temporal+P, 1024] or NULL,
 * vid_start [1]) into cache slot `slot` (0 <= slot < max_slots). The slot then holds positions
 * 0 .. S-1; no other slot's cache columns are read or written. next_tok [1] int32: the arg-max at the last
 * position. Like vcl_llm_prefill it clears the cache's left padding (vcl_llm_prefill_padded): the other slots
 * must be (re)started with vcl_llm_slot_prefill before they are decoded. */
int vcl_llm_slot_prefill(vcl_handle* h, int slot, const int64_t* ids, const void* video_feats,
                         const int32_t* vid_start, int S, int32_t* next_tok, void* stream);

/* Batched admission: n prompts into n cache slots in ONE pass of the layer stack. Prompt i has seq_len_host[i]
 * tokens and goes to slot slots_host[i] (both HOST memory, [n] int32). ids is the packed [sum S_i] int64: the
 * prompts concatenated without padding. video_feats is [n, n_temporal+P, 1024] or NULL; vid_start [n] int32 and
 * next_tok [n] int32 are device arrays, vid_start[i] counted from prompt i's first token (VCL_NO_VIDEO: prompt i
 * is text only and its feature rows are ignored). Every prompt comes out exactly as vcl_llm_slot_prefill of that
 * prompt alone leaves it: the same cache bits in its slot (columns 0 .. S_i-1) and the same first token
 * next_tok[i]. No other cache column is read or written. Like vcl_llm_slot_prefill it clears the cache's left
 * padding. Rejected before any device work, the handle and cache untouched: n outside 1 .. max_slots,
 * a slot outside 0 .. max_slots-1 or given twice, S_i outside 1 .. min(512, max_seq) (512: the key limit
 * of the prefill attention kernel). So sum S_i never exceeds the activations (max_batch * max_seq rows). The call always
 * runs the q|k|v GEMM's fused RoPE / cache-write epilogue and the wgmma prefill attention, whatever
 * VCL_PREFILL_ROPE_SEPARATE and VCL_PREFILL_ATTN_FLASH say (those switch the other prefill entry points only).
 * Its launches do not depend on n beyond the choice of decode kernel for the lm_head (1..4, 5..16 or 17..64 rows); the
 * row layout reaches the kernels through one host-to-device copy into a device map of the handle. */
int vcl_llm_slots_prefill(vcl_handle* h, int n, const int32_t* slots_host, const int32_t* seq_len_host,
                          const int64_t* ids, const void* video_feats, const int32_t* vid_start,
                          int32_t* next_tok, void* stream);

/* Chunked prefill on a PAGED cache (vcl_config.kv_blocks > 0; rejected otherwise): prompts longer than 512 tokens
 * run through the layer stack in chunks of at most 512 rows, each attending the cache columns its earlier chunks
 * left there. Sequence i is rows start_host[i] .. start_host[i] + len_host[i] - 1 of a prompt of total_host[i]
 * tokens in slot slots_host[i] (all HOST memory, [n] int32); columns 0 .. start_host[i] - 1 of that slot must hold
 * the prompt's earlier chunks. ids is the packed [sum len_i] int64 of the chunks. video_feats / vid_start are those
 * of vcl_llm_slots_prefill, vid_start[i] counted from the prompt's first token: row p of the prompt takes feature row
 * p - vid_start[i] - 1 when that lies in the span, so a span may straddle a chunk boundary. RoPE positions and cache
 * columns are absolute (start_i + j). The attention follows the contiguous engine's choice for the whole prompt:
 * total_i > 512 runs the mma.sync flash kernel of a one-shot prefill over more than 512 keys, with each key tile read
 * through the block table; total_i <= 512 needs start_i = 0 and len_i = total_i (vcl_llm_slots_prefill) and runs the
 * wgmma kernel; one launch per kernel kind present. So after the last chunk the slot's columns 0 .. total_i - 1 and
 * its first token equal vcl_llm_slot_prefill of the whole prompt on a contiguous handle, bit for bit, however the
 * prompt was cut. next_tok [n] int32: the token at each chunk's last row, drawn with entry slots_host[i] of the
 * sampling table at counter start_i + len_i (only the last chunk's token is the prompt's first token). Rejected
 * before any device work, the handle untouched: n outside 1 .. max_slots, a slot outside 0 .. max_slots-1 or given
 * twice, start_i not a multiple of 64, len_i outside 1 .. 512, start_i + len_i > total_i, total_i > max_seq, a
 * prompt of at most 512 tokens that is not whole, and sum len_i beyond the activations (max_batch * min(max_seq,
 * 512) rows). */
int vcl_llm_slots_prefill_chunk(vcl_handle* h, int n, const int32_t* slots_host, const int32_t* start_host,
                                const int32_t* len_host, const int32_t* total_host, const int64_t* ids,
                                const void* video_feats, const int32_t* vid_start, int32_t* next_tok, void* stream);

/* Continued prefill on a PAGED cache (vcl_config.kv_blocks > 0; rejected otherwise): vcl_llm_prefill_append for
 * several slots in one packed pass. Sequence i is the text-only tail of len_host[i] tokens at positions
 * start_host[i] .. start_host[i] + len_host[i] - 1 of slot slots_host[i] (all HOST memory, [n] int32), whose
 * columns 0 .. start_host[i] - 1 the slot already holds (a kept conversation: its prompt, the answer's decoded
 * columns). ids is the packed [sum len_i] int64 of the tails. Each tail runs the attention kernel the contiguous
 * continued prefill runs at the same start and length: the wgmma kernel when start_i + len_i <= 512, the flash kernel
 * otherwise, with the same tiles and masks (VCL_PREFILL_ATTN_FLASH does not apply); one launch per kernel kind
 * present. So the slot's columns start_i .. start_i + len_i - 1 and next_tok[i] equal vcl_llm_prefill_append(ids_i,
 * B = 1, S = len_i, start_pos = start_i) on a contiguous handle holding the same columns 0 .. start_i - 1, bit for
 * bit. next_tok [n] int32 is drawn with entry slots_host[i] of the sampling table at counter start_i + len_i.
 * Rejected before any device work, the handle untouched: n outside 1 .. max_slots, a slot outside 0 .. max_slots-1
 * or given twice, start_i < 1, len_i outside 1 .. 512, start_i + len_i > max_seq, and sum len_i beyond the
 * activations (max_batch * min(max_seq, 512) rows). */
int vcl_llm_slots_prefill_append(vcl_handle* h, int n, const int32_t* slots_host, const int32_t* start_host,
                                 const int32_t* len_host, const int64_t* ids, int32_t* next_tok, void* stream);

/* vcl_llm_decode_loop with a position per slot: slot b (0 <= b < n_slots) is fed first_tok[b] at position
 * pos_host[b] (HOST memory: the number of tokens its cache holds), then runs n_new-1 greedy steps;
 * out_tokens is [n_slots, n_new] int32, first_tok included. Every pos_host[b] + n_new - 1 must be <= max_seq
 * (checked before any device work). A slot without a request is computed like any other; its tokens are
 * meaningless and it writes only its own cache columns (park it at position 0). The positions are copied to
 * a device array of the handle at a fixed address, so one CUDA graph per (n_slots, n_new) serves every set of
 * positions; it is the graph vcl_llm_decode_loop uses for (B = n_slots, n_new). 1 <= n_slots <= max_slots;
 * a left-padded cache is rejected. */
int vcl_llm_slot_decode(vcl_handle* h, const int32_t* first_tok, const int32_t* pos_host, int n_slots, int n_new,
                        int32_t* out_tokens, void* stream);

/* Sampling (model.generate(do_sample=True, temperature=T, top_k=k), video_chatgpt/inference.py:105-107, i.e.
 * transformers' TemperatureLogitsWarper then TopKLogitsWarper then a multinomial draw). The handle holds one
 * sampling table of max_batch entries at fixed device addresses; entry b belongs to clip b, or to cache slot b.
 * Every call that produces a token (vcl_llm_prefill(_padded), _prefill_append, _decode_step, _generate(_padded),
 * _decode_loop, _slot_prefill, _slots_prefill -- prompt i with entry slots_host[i] -- and _slot_decode) picks
 * clip b's token by entry b: temperature 0 is greedy (the arg-max), otherwise the token is drawn from
 * softmax(logits / T) over the top-k logits (ties at the k-th value kept; k = 0 or k >= vocab keeps all) with
 * u from Philox4x32-10, key = the entry's seed, counter = the RoPE position the new token takes. So a sequence's
 * tokens depend on (seed, positions) only, not on its clip or slot, its neighbours, padding or chunking. A row
 * whose scaled maximum logit is not finite falls back to the arg-max. The exact rules are in DESIGN.md section 3.
 * When every entry a call uses is greedy, the call launches the same kernels as before any sampling was set; a
 * sampled decode loop has a CUDA graph of its own per (B, n_new), replayed for any settings.
 *
 * vcl_llm_set_sampling writes n entries: clip clips_host[i] gets temperature_host[i], top_k_host[i] and
 * seed_host[i] (all HOST memory, [n]); one host-to-device copy on `stream`. All entries are greedy after
 * vcl_create. Rejected before any device work: n outside 1 .. max_batch, a clip outside 0 .. max_batch-1 or
 * given twice, a temperature below 0 or not finite, a negative top_k. */
int vcl_llm_set_sampling(vcl_handle* h, int n, const int32_t* clips_host, const float* temperature_host,
                         const int32_t* top_k_host, const uint64_t* seed_host, void* stream);

/* Top-p (nucleus) sampling and the repetition penalty (HF's TopPLogitsWarper and RepetitionPenaltyLogitsProcessor,
 * in HF's order: penalty, temperature, top-k, top-p). vcl_llm_set_sampling_ex is vcl_llm_set_sampling plus, per
 * entry, top_p_host[i] (0 .. 1; 1 off) and repetition_penalty_host[i] (> 0; 1 off); vcl_llm_set_sampling itself sets
 * both to 1. The penalty applies to greedy and sampled entries: a logit x of a token in the entry's TOKEN SET becomes
 * x < 0 ? x * r : x / r (fp32) before the temperature. Top-p applies to sampled entries: of the tokens top-k keeps,
 * those whose mass strictly above them (fixed-point, in key order) is below top_p times the kept mass, ties whole
 * and the largest always kept; the draw and the log-probs then use that final set. The exact rules are in DESIGN.md
 * section 3. An entry with either setting takes a 32-bit sampler that adds the token it picks to the entry's token
 * set, so a decode loop keeps it current on the device; a call uses it when one of its entries has a penalty, or
 * samples with top_p < 1, and then launches it instead of the arg-max kernels (a sampled decode loop of these entries
 * has its own CUDA graph per (B, n_new)). Calls whose entries all have top_p 1 and penalty 1 launch what they
 * launched before. The first call that turns a penalty on allocates the token sets, one bitmap of ceil(vocab / 32)
 * int32 words per entry (256 KB at max_batch 64, vocab 32003). Rejected before any device work: what
 * vcl_llm_set_sampling rejects, a top_p outside [0, 1] or NaN, a penalty <= 0 or not finite, and either setting on
 * a vocabulary over VCL_SAMPLE_WIDE_MAX_V (the 32-bit sampler stages a row of 4-byte keys in shared memory). */
#define VCL_SAMPLE_WIDE_MAX_V 57344
int vcl_llm_set_sampling_ex(vcl_handle* h, int n, const int32_t* clips_host, const float* temperature_host,
                            const int32_t* top_k_host, const uint64_t* seed_host, const float* top_p_host,
                            const float* repetition_penalty_host, void* stream);

/* The token set of entry `entry` (HF's input_ids of its row: the prompt with its video placeholder and pad ids, then
 * every token generated so far; for a continued conversation the whole conversation): cleared, then ids[0 .. n)
 * (DEVICE int64; ids outside 0 .. vocab-1 are ignored) marked, in one kernel on `stream`. Set it before the call that
 * produces the entry's first token with a penalty; the sampler then adds each token it picks. Rejected before any
 * device work: an entry outside 0 .. max_batch-1, n < 0, null ids with n > 0, a vocabulary over
 * VCL_SAMPLE_WIDE_MAX_V. */
int vcl_llm_set_token_set(vcl_handle* h, int entry, const int64_t* ids, int n, void* stream);

/* Copy entry `entry`'s token set, ceil(vocab / 32) uint32 words (bit i & 31 of word i >> 5: token i), to bits_out
 * (host or device memory), ordered on `stream`. Rejected: a null argument, an entry outside 0 .. max_batch-1, a
 * handle that never allocated its token sets. */
int vcl_llm_read_token_set(vcl_handle* h, int entry, uint32_t* bits_out, void* stream);

/* Log-probabilities of generated tokens: what HF returns as generate(output_scores=True) followed by
 * compute_transition_scores(sequences, scores, normalize_logits=True) ($TF/generation/utils.py), plus the top-n
 * alternatives of each step, computed on the device by the sampler next to the token it picks. For the token of
 * an entry that asks, with s the processed scores HF's `scores` holds (greedy: the logits; sampled: logits / T over
 * the tokens top-k keeps, -inf elsewhere; a NaN logit is never kept), m = max s and W = sum of exp(s - m) over the
 * kept tokens (for a sampled row the sum the draw uses, in its order): lp(j) = (s_j - m) - logf(W). The exact rules
 * are in DESIGN.md section 3. A row's values depend on its logits row and its entry only.
 *
 * vcl_llm_set_logprobs writes n entries of the handle's sampling table: clip / slot clips_host[i] gets
 * top_n_host[i] (HOST memory, [n]): -1 off (every entry after vcl_create), 0 the chosen token only, 1 ..
 * VCL_LOGPROBS_MAX that many alternatives as well. One host-to-device copy on `stream`. Every token-producing call
 * (the list at vcl_llm_set_sampling, on a contiguous or a paged handle) then writes, for each entry that asks, 1 +
 * VCL_LOGPROBS_MAX pairs (int32 id, f32 lp) at (entry, RoPE position of the token) of a buffer the handle owns,
 * [max_batch][max_seq + 1][1 + VCL_LOGPROBS_MAX] ids and as many log-probs, allocated by the first call that turns an
 * entry on (22 MB at max_batch 64, max_seq 2048; a handle that never asks holds none). Place 0 is the chosen token; places 1 .. top_n
 * the top_n kept tokens of largest s (ties: lowest index), -1 / -inf where fewer are kept; a row without a finite
 * maximum (the arg-max fallback) has NaN everywhere and id -1 at places 1 .. top_n; places past top_n are not
 * written. A call whose entries are all greedy with log-probs off runs the kernels it ran before; otherwise the
 * sampler replaces the arg-max kernels, with the same tokens (a greedy entry's token is the arg-max either way).
 * Rejected before any device work: n outside 1 .. max_batch, a clip outside 0 .. max_batch-1 or given twice, a
 * top_n outside -1 .. VCL_LOGPROBS_MAX. */
#define VCL_LOGPROBS_MAX 20
int vcl_llm_set_logprobs(vcl_handle* h, int n, const int32_t* clips_host, const int32_t* top_n_host, void* stream);

/* Copy the log-prob rows of positions first_pos .. first_pos + count - 1 of entry `entry` out of the handle's buffer:
 * ids_out [count][1 + VCL_LOGPROBS_MAX] int32 and lp_out [count][1 + VCL_LOGPROBS_MAX] f32, host or device memory,
 * ordered on `stream`. The token generated at position p of entry b (a prefill of S tokens into clip b: p = S -
 * n_pad[b]; decode tokens follow at p + 1, ...) is row p. Rejected before any device work: a null argument, a handle
 * whose buffer was never allocated, an entry outside 0 .. max_batch-1, positions outside 0 .. max_seq. */
int vcl_llm_read_logprobs(vcl_handle* h, int entry, int first_pos, int count, int32_t* ids_out, float* lp_out,
                          void* stream);

/* Paged KV cache (vcl_config.kv_blocks > 0). The cache is a pool of kv_blocks BLOCKS. A block holds 128 cache columns
 * of one sequence across all layers, [layer][K = 0 | V = 1][head][128 columns][128 dims] bf16 (2 * llm_layers *
 * llm_heads * 32 KiB: 64 MiB at 7B, 100 MiB at 13B), one contiguous range. The BLOCK TABLE, int32
 * [n_slots][ceil(max_seq / 128)] with n_slots the slot count (max_slots, see above), maps column c of cache slot s to
 * block table[s][c / 128], offset c % 128. Block 0 is the PARK BLOCK: no sequence owns it, and every table entry
 * that no sequence owns points at it, so a parked slot (position 0) writes into it and into nothing else. Usable
 * capacity is kv_blocks - 1 blocks. The table starts all zeros. Every result is bit for bit that of the contiguous
 * cache: only the address of a column changes. The caller makes the table cover every column a call writes that
 * it will read again: a slot prefill of S tokens writes columns 0 .. S-1, a slot decode of n_new tokens at pos
 * writes pos .. pos + n_new - 2.
 *
 * A paged handle serves vcl_llm_slots_prefill, vcl_llm_slot_prefill (run as a packed prefill of one prompt, so
 * prompts are limited to min(512, max_seq) tokens), vcl_llm_slots_prefill_chunk (prompts up to max_seq tokens, in
 * chunks of at most 512 rows), vcl_llm_slots_prefill_append (text tails of kept conversations), vcl_llm_slot_decode and vcl_llm_set_sampling. Every static
 * entry point (vcl_llm_prefill(_padded, _states, _append), _decode_step, _decode_loop, _generate(_padded), _score)
 * and vcl_kv_cache_copy is rejected. Its LLM activations are sized for max_batch * min(max_seq, 512) rows, the
 * most a packed prefill uses.
 *
 * vcl_llm_set_block_table writes the whole table from table_host (HOST memory, n_slots * ceil(max_seq / 128)
 * int32, row-major) with one host-to-device copy on `stream` into a device array of the handle at a fixed address,
 * so one captured slot-decode graph serves every table. Rejected before any device work, the table unchanged: an
 * entry outside 0 .. kv_blocks-1, or a block other than 0 that appears twice. Not a paged handle: rejected. */
int vcl_llm_set_block_table(vcl_handle* h, const int32_t* table_host, void* stream);

/* Copy block `block` (0 .. kv_blocks-1) of a paged cache whole out of the handle into buf (write = 0) or from buf
 * into it (write = 1): one cudaMemcpyAsync on `stream`. buf is device memory or pinned host memory of the block's
 * size (above). Swapping a sequence out to host memory and back, and reading the cache back in tests. */
int vcl_kv_block_copy(vcl_handle* h, int block, int write, void* buf, void* stream);

/* forward(input_ids, labels=..., ...) (video_chatgpt/model/video_chatgpt.py:225-239): lm_head at EVERY
 * position and, with labels, the shifted cross-entropy of CrossEntropyLoss (ignore_index -100): column s of
 * clip b is scored against labels[b, s+1]; column S-1 has no target. The prefill is vcl_llm_prefill's
 * (n_pad_host NULL) or vcl_llm_prefill_padded's (n_pad_host as there), and leaves the KV cache, and its
 * padding state, exactly as that call does, so cached steps can follow.
 *   labels      optional [B,S] int64; -100 is not scored. A label outside 0 .. vocab-1 gives a NaN row (and a
 *               NaN loss); it is never used as an index
 *   logits_out  optional [B,S,vocab] bf16: every position's logits, as the reference's logits tensor
 *   nll_out     optional [B,S-1] fp32 (needs labels): -log_softmax(logits[b,s])[labels[b,s+1]], the
 *               log-softmax computed in fp32 and rounded to bf16 as torch does on bf16 logits; 0 where the
 *               label is -100
 *   loss_out    optional [1] fp32 (needs labels): the mean of nll over the scored positions (NaN when
 *               there is none, as in torch); fixed summation order, identical from run to run
 * Work space is the handle's activation buffers: the lm_head GEMM runs over chunks of rows that fit the
 * q|k|v activation (max_batch * max_seq * 3 * llm_hidden elements). */
int vcl_llm_score(vcl_handle* h, const int64_t* ids, const void* video_feats, const int32_t* vid_start,
                  const int32_t* n_pad_host, int B, int S, const int64_t* labels, void* logits_out, float* nll_out,
                  float* loss_out, void* stream);

/* Number of kernels of this library launched so far in the process (CUDA-graph replays count the
 * kernel nodes they contain). Evidence for bench.py's "gpu_launches". */
long long vcl_launch_count(void);

/* ---- single-operator entry points (unit tests / profiling of the individual kernels) ---- */
/* C[M,N] = act(A[M,K] . W[N,K]^T + bias) (+ residual); act: 0 none, 1 quick_gelu, 2 gelu(erf),
 * 3 swiglu over interleaved rows (C is [M,N/2]). block_n: 0 = auto, or 32/64/128/256. */
int vcl_op_gemm(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc,
                const void* bias, const void* residual, int64_t ldr, int M, int N, int K, int act,
                int block_n, void* stream);
/* same with an explicit thread-block-cluster size along M (1, 2 or 4): the CTAs of a cluster share
 * each weight tile through TMA multicast (block_n 128 or 256; narrower tiles run without a cluster);
 * cluster = -2: a CTA pair on one 256-row tile, each CTA fetching half of the weight tile (on sm_90 the same
 * launch as cluster = 2, since a wgmma reads only its own CTA's shared memory) */
int vcl_op_gemm_ex(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc,
                   const void* bias, const void* residual, int64_t ldr, int M, int N, int K, int act,
                   int block_n, int cluster, void* stream);
/* The cross-entropy kernel of vcl_llm_score without the shift: logits [rows, ld] bf16 (first V columns
 * used; 16-byte aligned, ld a multiple of 8), labels [rows] int64 (-100 ignored) -> nll_out [rows] fp32
 * (required) and, optionally, loss_out [1] fp32, the mean over the rows whose label is not -100. */
int vcl_op_cross_entropy(const void* logits, int64_t ld, const int64_t* labels, int rows, int V,
                         float* nll_out, float* loss_out, void* stream);
/* The sampling kernel on its own: row b of logits [B, ld] fp32 (first V columns; bf16-representable values, as
 * the lm_head writes them) is sampled with temperature_host[b] (0: greedy), top_k_host[b], seed_host[b] and the
 * Philox counter counter_host[b] (all HOST memory, [B]); tok_out [B] int32 on the device. V <= 81920. */
int vcl_op_sample(const float* logits, int64_t ld, int B, int V, const float* temperature_host,
                  const int32_t* top_k_host, const uint64_t* seed_host, const int32_t* counter_host, int32_t* tok_out,
                  void* stream);
/* vcl_op_sample with log-probs (compute_transition_scores(normalize_logits=True) on HF's output_scores, and the
 * top-n alternatives; see vcl_llm_set_logprobs): row b also writes places 0 .. top_n_host[b] (HOST memory, [B],
 * -1 .. VCL_LOGPROBS_MAX; -1 writes none) of ids_out / lp_out [B][1 + VCL_LOGPROBS_MAX] (device int32 / f32).
 * tok_out equals vcl_op_sample's bit for bit. */
int vcl_op_sample_logprobs(const float* logits, int64_t ld, int B, int V, const float* temperature_host,
                           const int32_t* top_k_host, const uint64_t* seed_host, const int32_t* counter_host,
                           const int32_t* top_n_host, int32_t* tok_out, int32_t* ids_out, float* lp_out,
                           void* stream);
/* The 32-bit sampler on its own (vcl_llm_set_sampling_ex): vcl_op_sample with top_p_host[b] and
 * repetition_penalty_host[b] (HOST memory, [B]), token_sets [B][ceil(V / 32)] uint32 on the device (null: every
 * set empty; row b's picked token is added to its set) and, when top_n_host is not null, vcl_op_sample_logprobs'
 * log-probs. A row with top_p 1 and penalty 1 gives vcl_op_sample(_logprobs)'s token and values bit for bit.
 * V <= VCL_SAMPLE_WIDE_MAX_V. */
int vcl_op_sample_ex(const float* logits, int64_t ld, int B, int V, const float* temperature_host,
                     const int32_t* top_k_host, const uint64_t* seed_host, const int32_t* counter_host,
                     const float* top_p_host, const float* repetition_penalty_host, uint32_t* token_sets,
                     const int32_t* top_n_host, int32_t* tok_out, int32_t* ids_out, float* lp_out, void* stream);
int vcl_op_layernorm(const void* x, void* y, const void* w, const void* b, int rows, int D, float eps,
                     void* stream);
int vcl_op_rmsnorm(const void* x, void* y, const void* w, int rows, int D, float eps, void* stream);
/* q,k,v,o: [B,S,H,hd] contiguous bf16 */
int vcl_op_attention(const void* q, const void* k, const void* v, void* o, int B, int S, int H,
                     int head_dim, float scale, int causal, void* stream);
/* ViT attention on the fused projection output: qkv [n_frames*S, 3*H*64] (q|k|v) -> out
 * [n_frames*S, H*64]; non-causal, scale 64^-1/2; wgmma kernel for 129 <= S <= 257 */
int vcl_op_attention_vit(const void* qkv, void* out, int n_frames, int S, int H, void* stream);
/* Copy decoder layer `layer`'s whole K and V cache, each [max_batch][llm_heads][max_seq][128] bf16, out of the
 * handle into k / v (write = 0) or from k / v into the handle (write = 1): one cudaMemcpyAsync per tensor on
 * `stream`. Lets a test read back exactly what the RoPE / cache writers stored, or fill the cache with a sentinel
 * first to see which columns a call touches. A paged handle (vcl_config.kv_blocks > 0) rejects it: see
 * vcl_kv_block_copy. */
int vcl_kv_cache_copy(vcl_handle* h, int layer, int write, void* k, void* v, void* stream);
/* The decode attention kernel on its own: q [B][q_ld] (head h at columns h*128 ..), k / v caches
 * [B][H][s_max][128], clip b's query at column c_b = kv_len - 1 + (pos_dev ? pos_dev[b] : 0) attending keys
 * n_pad[b] .. c_b (pos_dev, n_pad: device int32 [B]; pos_dev may be NULL). o [B][H*128] row-major, or with
 * o_xwin the window-major layout of the 5..16-clip decode kernels (kernels.h: xwin_offset, a buffer of
 * ceil(H*128 / 512) * B * 544 elements). With pos_dev, shared memory is sized for s_max keys. */
int vcl_op_decode_attention(const void* q, int64_t q_ld, const void* k, const void* v, void* o, int B, int H,
                            int s_max, int kv_len, const int32_t* pos_dev, const int32_t* n_pad, float scale,
                            int o_xwin, void* stream);
/* out[b,n] = x[b,:].W[n,:] (+res) with optional RMSNorm of x: B <= 4 the ring kernel of the single-clip
 * decode path (fused norm), 5 <= B <= 16 the wide ring kernel (norm + window-major re-layout by a launch of
 * its own, as on the decode path) */
int vcl_op_gemv(const void* x, const void* W, void* out, const void* res, const void* norm_w,
                float eps, int B, int N, int K, void* stream);
/* The load-time quantizer of VCL_WEIGHTS_FP8_E4M3 on its own, rows in order: W [N,K] bf16 (K a multiple of 32)
 * -> w_deq [N,K] bf16 = W~ (may be W), scales [N] fp32 = 2^e_r, codes = ceil(N/16)*16*K bytes in the slot order of
 * the decode kernels: row r, column k at (r/16)*16*K + (k/512)*8192 + (k%512/32)*512 + (r%16/8)*256 +
 * ((r%8)*4 + k%32/8)*8 + k%8 (rows past N zero). Nothing is checked: a non-finite row gives unspecified codes. */
int vcl_op_quantize_fp8(const void* W, int N, int K, void* w_deq, void* codes, float* scales, void* stream);
/* vcl_op_gemv with fp8 weights: W is quantized by the quantizer above (into scratch; W is not changed) and the
 * fp8 instances of the ring kernels run; equals vcl_op_gemv on W~ bit for bit. */
int vcl_op_gemv_fp8(const void* x, const void* W, void* out, const void* res, const void* norm_w,
                    float eps, int B, int N, int K, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VCL_H_ */

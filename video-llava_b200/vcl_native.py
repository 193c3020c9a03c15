"""ctypes binding of libvcl.so (include/vcl.h). PyTorch is used only as the owner of device
memory and streams: every call passes raw device pointers and the current CUDA stream.

There is no fallback: if the shared library is missing or the device is not an sm_90 (H100) GPU the
calls raise.
"""
from __future__ import annotations

import ctypes
import operator
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_uint64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvcl.so")

DTYPE_F16, DTYPE_BF16 = 0, 1
PIXELS_BF16_NCHW, PIXELS_U8_NHWC = 0, 1
RESIZE_MODES = {"nearest": 0, "bicubic": 1}   # VCL_RESIZE_NEAREST (load_video's torch rule), VCL_RESIZE_BICUBIC (PIL's)
PROJ_LINEAR, PROJ_MLP2X_GELU = 0, 1
NO_VIDEO = -2 ** 31          # vid_start value of a text-only row (VCL_NO_VIDEO)
ACT_NONE, ACT_QGELU, ACT_GELU, ACT_SWIGLU = 0, 1, 2, 3
WEIGHTS_BF16, WEIGHTS_FP8_E4M3 = 0, 1
WEIGHT_FORMATS = {"bf16": WEIGHTS_BF16, "fp8_e4m3": WEIGHTS_FP8_E4M3}   # the language model's weight formats


def weight_format_code(name) -> int:
    """"bf16" | "fp8_e4m3" -> VCL_WEIGHTS_*; anything else raises ValueError."""
    if not isinstance(name, str) or name not in WEIGHT_FORMATS:
        raise ValueError(f"unknown LLM weight format {name!r}: one of {sorted(WEIGHT_FORMATS)}")
    return WEIGHT_FORMATS[name]


class VclError(RuntimeError):
    pass


class vcl_config(Structure):
    _fields_ = [
        ("clip_layers", c_int32), ("clip_hidden", c_int32), ("clip_inter", c_int32),
        ("clip_heads", c_int32), ("image_size", c_int32), ("patch_size", c_int32),
        ("clip_ln_eps", c_float),
        ("llm_layers", c_int32), ("llm_hidden", c_int32), ("llm_inter", c_int32),
        ("llm_heads", c_int32), ("vocab", c_int32), ("rms_eps", c_float), ("rope_theta", c_float),
        ("proj_type", c_int32), ("n_temporal", c_int32),
        ("max_frames", c_int32), ("max_batch", c_int32), ("max_seq", c_int32),
        ("max_slots", c_int32),    # 0: min(max_batch, 16) in-flight cache slots
    ]


class vcl_config_ex(vcl_config):
    """The whole C vcl_config: the fields above, then the trailing kv_blocks (0: the contiguous KV cache; > 0: a paged
    cache of that many 128-column blocks). Engine always passes this struct to vcl_create; a plain vcl_config is
    copied into one, with kv_blocks from Engine's argument."""
    _fields_ = [("kv_blocks", c_int32)]


KV_BLOCK_COLS = 128          # cache columns per block of a paged KV cache


def kv_block_bytes(llm_layers: int, llm_heads: int) -> int:
    """Bytes of one block of a paged KV cache: [layer][K | V][head][128 columns][128 dims] bf16"""
    return 2 * int(llm_layers) * int(llm_heads) * KV_BLOCK_COLS * 128 * 2


def check_kv_blocks(kv_blocks):
    """kv_blocks of a paged cache -> int (None -> 0, the contiguous cache). Raises ValueError for anything else than
    None or an int >= 2 (block 0 is the park block)."""
    if kv_blocks is None:
        return 0
    try:
        n = None if isinstance(kv_blocks, bool) else operator.index(kv_blocks)
    except TypeError:
        n = None
    if n is None or n < 2:
        raise ValueError(f"kv_blocks={kv_blocks!r}: None (contiguous cache) or an int >= 2 (block 0 is the park block)")
    return n


def slot_capacity(max_batch: int, max_slots=None) -> int:
    """The engine's in-flight cache slots: max_slots, or min(max_batch, 16) for None. Raises ValueError for any
    other value outside 1 .. min(max_batch, 64) (vcl_create would reject it; its 0 is spelled None here)."""
    if max_slots is None:
        return min(int(max_batch), 16)
    try:
        n = None if isinstance(max_slots, bool) else operator.index(max_slots)     # int, numpy integers
    except TypeError:
        n = None
    if n is None or not 1 <= n <= min(int(max_batch), 64):
        raise ValueError(f"max_slots={max_slots!r} outside 1..{min(int(max_batch), 64)} (at most 64 and at most "
                         f"max_batch {max_batch}; None: min(max_batch, 16))")
    return n


class vcl_tensor(Structure):
    _fields_ = [("name", c_char_p), ("data", c_void_p), ("ndim", c_int32), ("shape", c_int64 * 4)]


# name -> (restype, argtypes); mirrors include/vcl.h one to one
_SIGNATURES = {
    "vcl_version": (c_int, []),
    "vcl_last_error": (c_char_p, []),
    "vcl_create": (c_int, [POINTER(c_void_p), POINTER(vcl_config)]),
    "vcl_destroy": (None, [c_void_p]),
    "vcl_load_clip_weights": (c_int, [c_void_p, POINTER(vcl_tensor), c_int]),
    "vcl_load_llm_weights": (c_int, [c_void_p, POINTER(vcl_tensor), c_int]),
    "vcl_load_llm_weights_ex": (c_int, [c_void_p, POINTER(vcl_tensor), c_int, c_int]),
    "vcl_clip_encode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "vcl_st_pool": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                            c_int, c_void_p]),
    "vcl_clip_features": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "vcl_resize_frames_workspace_bytes": (ctypes.c_size_t, [c_int] * 10),
    "vcl_resize_frames": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                  c_void_p, c_void_p, ctypes.c_size_t, c_void_p]),
    "vcl_llm_prefill": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p,
                                c_void_p, c_void_p, c_void_p]),
    "vcl_llm_prefill_states": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_prefill_append": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_decode_step": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_generate": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p,
                                 c_void_p]),
    "vcl_llm_decode_loop": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "vcl_llm_prefill_padded": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int32), c_int, c_int, c_int,
                                       c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_generate_padded": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int32), c_int, c_int, c_int,
                                        c_void_p, c_void_p]),
    "vcl_llm_score": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int32), c_int, c_int, c_void_p,
                              c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_slot_prefill": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "vcl_llm_slots_prefill": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int32), c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "vcl_llm_slots_prefill_chunk": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int32), POINTER(c_int32),
                                            POINTER(c_int32), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_slots_prefill_append": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int32), POINTER(c_int32),
                                             c_void_p, c_void_p, c_void_p]),
    "vcl_llm_slots_fork": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int32), POINTER(c_int32), c_void_p]),
    "vcl_llm_slots_score_append": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int32), POINTER(c_int32),
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_slot_decode": (c_int, [c_void_p, c_void_p, POINTER(c_int32), c_int, c_int, c_void_p, c_void_p]),
    "vcl_llm_set_sampling": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_float), POINTER(c_int32),
                                     POINTER(c_uint64), c_void_p]),
    "vcl_llm_set_sampling_ex": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_float), POINTER(c_int32),
                                        POINTER(c_uint64), POINTER(c_float), POINTER(c_float), c_void_p]),
    "vcl_llm_set_warpers": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_float), POINTER(c_float),
                                    POINTER(c_float), POINTER(c_float), c_void_p]),
    "vcl_llm_set_token_set": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "vcl_llm_read_token_set": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "vcl_llm_set_bans": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int32), POINTER(c_int32),
                                 POINTER(c_int32), POINTER(c_int32), c_void_p]),
    "vcl_llm_set_token_history": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "vcl_llm_read_token_history": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "vcl_llm_set_logprobs": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int32), c_void_p]),
    "vcl_llm_read_logprobs": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_set_guidance": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_int32), POINTER(c_float), c_void_p]),
    "vcl_llm_beam_start": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int32), c_int, c_int, c_int, c_int,
                                   c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_beam_decode": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_contrastive_start": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int32), c_int, c_int,
                                          c_int, c_float, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_contrastive_decode": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_launch_count": (ctypes.c_longlong, []),
    "vcl_kv_cache_copy": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_llm_set_block_table": (c_int, [c_void_p, POINTER(c_int32), c_void_p]),
    "vcl_kv_block_copy": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "vcl_op_decode_attention": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                        c_void_p, c_void_p, c_float, c_int, c_void_p]),
    "vcl_op_decode_attention_paged": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                              c_int, c_void_p, c_void_p, c_float, c_int, POINTER(c_int32), c_int,
                                              c_int64, c_void_p]),
    "vcl_op_attention_cached": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                        c_int, POINTER(c_int32), c_void_p]),
    "vcl_op_attention_packed": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                        POINTER(c_int32), POINTER(c_int32), POINTER(c_int32), POINTER(c_int32),
                                        POINTER(c_int32), c_int, c_int, c_int64, c_void_p]),
    "vcl_op_cross_entropy": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_op_label_logprobs": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_op_attention_appended": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                          POINTER(c_int32), POINTER(c_int32), POINTER(c_int32), c_void_p]),
    "vcl_op_gemm": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p,
                            c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "vcl_op_gemm_ex": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p,
                               c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "vcl_op_sample": (c_int, [c_void_p, c_int64, c_int, c_int, POINTER(c_float), POINTER(c_int32), POINTER(c_uint64),
                              POINTER(c_int32), c_void_p, c_void_p]),
    "vcl_op_sample_bans": (c_int, [c_void_p, c_int64, c_int, c_int, POINTER(c_float), POINTER(c_int32),
                                   POINTER(c_uint64), POINTER(c_int32), POINTER(c_float), POINTER(c_float), c_void_p,
                                   c_void_p, c_int64, POINTER(c_int32), POINTER(c_int32), POINTER(c_int32),
                                   POINTER(c_int32), POINTER(c_int32), c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_op_sample_logprobs": (c_int, [c_void_p, c_int64, c_int, c_int, POINTER(c_float), POINTER(c_int32),
                                       POINTER(c_uint64), POINTER(c_int32), POINTER(c_int32), c_void_p, c_void_p,
                                       c_void_p, c_void_p]),
    "vcl_op_sample_ex": (c_int, [c_void_p, c_int64, c_int, c_int, POINTER(c_float), POINTER(c_int32), POINTER(c_uint64),
                                 POINTER(c_int32), POINTER(c_float), POINTER(c_float), c_void_p, POINTER(c_int32),
                                 c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_op_sample_warpers": (c_int, [c_void_p, c_int64, c_int, c_int, POINTER(c_float), POINTER(c_int32),
                                      POINTER(c_uint64), POINTER(c_int32), POINTER(c_float), POINTER(c_float), c_void_p,
                                      POINTER(c_float), POINTER(c_float), POINTER(c_float), POINTER(c_float),
                                      POINTER(c_int32), c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_op_guidance": (c_int, [c_void_p, c_int64, c_int, c_int, POINTER(c_int32), POINTER(c_float), c_void_p,
                                c_void_p]),
    "vcl_op_beam_select": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                   c_void_p]),
    "vcl_op_contrastive_rank": (c_int, [c_void_p, c_int64, POINTER(c_int32), c_int, c_int, c_int, c_int, c_void_p,
                                        c_void_p, c_void_p, c_float, c_void_p, c_void_p]),
    "vcl_op_layernorm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "vcl_op_rmsnorm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "vcl_op_im2col": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "vcl_op_clip_embed_ln": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                     c_float, c_void_p]),
    "vcl_op_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                 c_float, c_int, c_void_p]),
    "vcl_op_attention_vit": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "vcl_op_gemv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int,
                            c_int, c_void_p]),
    "vcl_op_gemv_fp8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int,
                                c_int, c_void_p]),
    "vcl_op_quantize_fp8": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "vcl_op_gemv_ex": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_float, c_int, c_int, c_int, c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


def lib() -> ctypes.CDLL:
    """Load libvcl.so (built in-tree by build.py). Fails loudly if it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VclError(f"{LIB_PATH} is missing: run `python video-llava_b200/build.py` "
                           "(there is no CPU or PyTorch fallback for this path)")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise VclError(f"libvcl error {rc}: {lib().vcl_last_error().decode()}")


def ptr(t) -> c_void_p:
    if t is None:
        return c_void_p(0)
    assert t.is_cuda and t.is_contiguous(), "vcl needs contiguous CUDA tensors"
    return c_void_p(t.data_ptr())


def cur_stream() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def _dtype_code(dt: torch.dtype) -> int:
    if dt == torch.float16:
        return DTYPE_F16
    if dt == torch.bfloat16:
        return DTYPE_BF16
    raise VclError(f"unsupported dtype {dt} (fp16 / bf16 only)")


# ---------------------------------------------------------------------------------------------
# stateless operators
# ---------------------------------------------------------------------------------------------
def st_pool(features: torch.Tensor, n_temporal: int = 100, out_dtype: torch.dtype = torch.float16):
    """[T,P,C] (fp16|bf16, last dim contiguous) -> [n_temporal+P, C]; see vcl_st_pool."""
    T, P, C = features.shape
    assert features.is_cuda and features.stride(2) == 1
    out = torch.empty(n_temporal + P, C, dtype=out_dtype, device=features.device)
    check(lib().vcl_st_pool(c_void_p(features.data_ptr()), _dtype_code(features.dtype),
                            features.stride(0), features.stride(1), T, P, C, n_temporal,
                            ptr(out), _dtype_code(out_dtype), cur_stream()))
    return out


def resize_frames(frames: torch.Tensor, size, mode: str, crop=None) -> torch.Tensor:
    """Resize raw frames on the device (vcl_resize_frames): frames uint8 [T,H,W,3] CUDA -> the frames resized to
    size = (h, w) with mode "nearest" (torch.nn.functional.interpolate's rule, as load_video) or "bicubic" (PIL's
    BICUBIC, as CLIPImageProcessor), then cut to crop = (top, left, crop_h, crop_w) (default: the whole frame):
    uint8 [T, crop_h, crop_w, 3], bit for bit what the CPU resize gives."""
    if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
        raise VclError("resize_frames: frames must be a uint8 [T,H,W,3] tensor, got "
                       f"{getattr(frames, 'dtype', type(frames))} {tuple(getattr(frames, 'shape', ()))}")
    if not frames.is_cuda:
        raise VclError("resize_frames: frames must live on the GPU (no CPU fallback)")
    if mode not in RESIZE_MODES:
        raise VclError(f"resize_frames: unknown mode {mode!r}: one of {sorted(RESIZE_MODES)}")
    frames = frames.contiguous()
    n, in_h, in_w = frames.shape[:3]
    out_h, out_w = (int(v) for v in size)
    top, left, crop_h, crop_w = (0, 0, out_h, out_w) if crop is None else (int(v) for v in crop)
    geo = (n, in_h, in_w, RESIZE_MODES[mode], out_h, out_w, top, left, crop_h, crop_w)
    ws_bytes = lib().vcl_resize_frames_workspace_bytes(*geo)
    if ws_bytes == ctypes.c_size_t(-1).value:
        raise VclError(f"libvcl error: {lib().vcl_last_error().decode()}")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=frames.device) if ws_bytes else None
    out = torch.empty(n, crop_h, crop_w, 3, dtype=torch.uint8, device=frames.device)
    check(lib().vcl_resize_frames(ptr(frames), *geo, ptr(out), ptr(ws), ws_bytes, cur_stream()))
    return out


def op_gemm(a, w, bias=None, residual=None, act=ACT_NONE, block_n=0, out=None, cluster=0):
    M, K = a.shape
    N = w.shape[0]
    n_out = N // 2 if act == ACT_SWIGLU else N
    if out is None:
        out = torch.empty(M, n_out, dtype=torch.bfloat16, device=a.device)
    check(lib().vcl_op_gemm_ex(ptr(a), a.stride(0), ptr(w), w.stride(0), ptr(out), out.stride(0), ptr(bias),
                               ptr(residual), residual.stride(0) if residual is not None else 0, M, N, K,
                               act, block_n, cluster, cur_stream()))
    return out


def op_layernorm(x, w, b, eps):
    y = torch.empty_like(x)
    check(lib().vcl_op_layernorm(ptr(x), ptr(y), ptr(w), ptr(b), x.shape[0], x.shape[1], eps, cur_stream()))
    return y


def op_rmsnorm(x, w, eps):
    y = torch.empty_like(x)
    check(lib().vcl_op_rmsnorm(ptr(x), ptr(y), ptr(w), x.shape[0], x.shape[1], eps, cur_stream()))
    return y


def op_attention(q, k, v, scale, causal):
    """q,k,v: [B,S,H,hd] contiguous bf16."""
    B, S, H, hd = q.shape
    o = torch.empty_like(q)
    check(lib().vcl_op_attention(ptr(q), ptr(k), ptr(v), ptr(o), B, S, H, hd, scale, int(causal), cur_stream()))
    return o


def op_im2col(pixels, fmt, KP, patch=14, out=None):
    """The patch gather alone (vcl_op_im2col): pixels [N,3,I,I] bf16 (fmt PIXELS_BF16_NCHW) or [N,I,I,3] uint8
    (PIXELS_U8_NHWC) -> [N * (I / patch)^2, KP] bf16 (out if given)."""
    n, image = pixels.shape[0], pixels.shape[2]
    P = (image // patch) ** 2
    if out is None:
        out = torch.empty(n * P, KP, dtype=torch.bfloat16, device=pixels.device)
    check(lib().vcl_op_im2col(ptr(pixels), fmt, ptr(out), n, image, patch, KP, cur_stream()))
    return out


def op_clip_embed_ln(patch_out, cls, pos, w, b, n_frames, eps, out=None):
    """The CLIP embedding + pre-LN alone (vcl_op_clip_embed_ln): patch_out [n_frames * P, D], cls [D], pos [P + 1, D],
    w / b [D], all bf16 -> h [n_frames * (P + 1), D] bf16 (out if given)."""
    D = cls.shape[-1]
    P = pos.shape[0] - 1
    if out is None:
        out = torch.empty(n_frames * (P + 1), D, dtype=torch.bfloat16, device=cls.device)
    check(lib().vcl_op_clip_embed_ln(ptr(patch_out), ptr(cls), ptr(pos), ptr(w), ptr(b), ptr(out), n_frames, P, D, eps,
                                     cur_stream()))
    return out


def op_attention_vit(qkv, n_frames, S, H, out=None):
    """qkv: [n_frames*S, 3*H*64] bf16 -> [n_frames*S, H*64] (ViT attention; out if given)."""
    if out is None:
        out = torch.empty(n_frames * S, H * 64, dtype=torch.bfloat16, device=qkv.device)
    check(lib().vcl_op_attention_vit(ptr(qkv), ptr(out), n_frames, S, H, cur_stream()))
    return out


def op_cross_entropy(logits, labels, V=None, want_loss=True):
    """logits [rows, ld] bf16 (the first V columns, default all; row pitch a multiple of 8), labels [rows] int64
    (-100 ignored) -> (nll [rows] fp32, loss 0-d fp32 | None); see vcl_op_cross_entropy."""
    rows, ld = logits.shape
    assert logits.dtype == torch.bfloat16 and logits.stride(1) == 1
    lab = labels.to(device=logits.device, dtype=torch.int64).contiguous()
    nll = torch.empty(rows, dtype=torch.float32, device=logits.device)
    loss = torch.empty((), dtype=torch.float32, device=logits.device) if want_loss else None
    check(lib().vcl_op_cross_entropy(c_void_p(logits.data_ptr()), logits.stride(0), ptr(lab), rows,
                                     ld if V is None else V, ptr(nll), ptr(loss), cur_stream()))
    return nll, loss


def op_label_logprobs(logits, labels, V=None):
    """The scoring kernel of candidate scoring alone (vcl_op_label_logprobs): logits [rows, ld] bf16 (the first V
    columns, default all), labels [rows] int64 -> (lp [rows] fp32, greedy [rows] bool) on the device: the greedy
    log-prob rule at each label, and whether it is the lowest-index arg-max of its row."""
    rows, ld = logits.shape
    assert logits.dtype == torch.bfloat16 and logits.stride(1) == 1
    lab = labels.to(device=logits.device, dtype=torch.int64).contiguous()
    lp = torch.empty(rows, dtype=torch.float32, device=logits.device)
    greedy = torch.empty(rows, dtype=torch.uint8, device=logits.device)
    check(lib().vcl_op_label_logprobs(c_void_p(logits.data_ptr()), logits.stride(0), rows, ld if V is None else V,
                                      ptr(lab), ptr(lp), ptr(greedy), cur_stream()))
    return lp, greedy.bool()


def _seeds(seeds, n):
    """n 64-bit seeds (ints, taken mod 2**64) -> ctypes uint64[n]"""
    vals = [int(v) % 2 ** 64 for v in seeds]
    if len(vals) != n:
        raise VclError(f"{len(vals)} seeds for {n} rows")
    return (c_uint64 * n)(*vals)


def op_sample(logits, temperature, top_k, seed, counter):
    """The sampling kernel alone (vcl_op_sample). logits [B, ld] fp32 on the device (bf16-representable values);
    temperature / top_k / seed / counter: B host values per row (temperature 0: greedy). Returns [B] int32."""
    B, ld = logits.shape
    assert logits.dtype == torch.float32 and logits.stride(1) == 1
    out = torch.empty(B, dtype=torch.int32, device=logits.device)
    vals = [list(v) for v in (temperature, top_k, counter)]
    if not all(len(v) == B for v in vals):
        raise VclError(f"temperature / top_k / counter need {B} entries each")
    check(lib().vcl_op_sample(c_void_p(logits.data_ptr()), logits.stride(0), B, ld,
                              (c_float * B)(*[float(t) for t in vals[0]]), (c_int32 * B)(*[int(k) for k in vals[1]]),
                              _seeds(seed, B), (c_int32 * B)(*[int(c) for c in vals[2]]), ptr(out), cur_stream()))
    return out


LOGPROBS_MAX = 20              # include/vcl.h: VCL_LOGPROBS_MAX, the most alternatives per token
LOGPROB_PLACES = 1 + LOGPROBS_MAX


def op_sample_logprobs(logits, temperature, top_k, seed, counter, top_n):
    """The sampling kernel with log-probs (vcl_op_sample_logprobs): op_sample's arguments plus top_n, B host ints
    (-1 .. LOGPROBS_MAX). Returns (tokens [B] int32, ids [B, LOGPROB_PLACES] int32, lp [B, LOGPROB_PLACES] f32) on
    the device: place 0 the chosen token, places 1 .. top_n[b] the alternatives; places past top_n[b] are -1 / NaN."""
    B, ld = logits.shape
    assert logits.dtype == torch.float32 and logits.stride(1) == 1
    vals = [list(v) for v in (temperature, top_k, counter, top_n)]
    if not all(len(v) == B for v in vals):
        raise VclError(f"temperature / top_k / counter / top_n need {B} entries each")
    out = torch.empty(B, dtype=torch.int32, device=logits.device)
    ids = torch.full((B, LOGPROB_PLACES), -1, dtype=torch.int32, device=logits.device)
    lp = torch.full((B, LOGPROB_PLACES), float("nan"), dtype=torch.float32, device=logits.device)
    ints = lambda v: (c_int32 * B)(*[int(x) for x in v])   # noqa: E731
    check(lib().vcl_op_sample_logprobs(c_void_p(logits.data_ptr()), logits.stride(0), B, ld,
                                       (c_float * B)(*[float(t) for t in vals[0]]), ints(vals[1]), _seeds(seed, B),
                                       ints(vals[2]), ints(vals[3]), ptr(out), ptr(ids), ptr(lp), cur_stream()))
    return out, ids, lp


SAMPLE_WIDE_MAX_V = 57344     # include/vcl.h: VCL_SAMPLE_WIDE_MAX_V, the vocabulary limit of top_p / repetition_penalty


def token_set_words(V):
    """int32 words of one token-set bitmap over a vocabulary of V tokens"""
    return (V + 31) // 32


def op_sample_ex(logits, temperature, top_k, seed, counter, top_p, repetition_penalty, token_sets=None, top_n=None):
    """The 32-bit sampler alone (vcl_op_sample_ex): op_sample's arguments plus top_p and repetition_penalty (B host
    values each), token_sets (None, or [B, token_set_words(V)] int32 on the device; each row's picked token is added
    to it) and top_n (None, or B host ints as in op_sample_logprobs). Returns tokens [B] int32, or (tokens, ids, lp)
    with top_n."""
    B, ld = logits.shape
    assert logits.dtype == torch.float32 and logits.stride(1) == 1
    vals = [list(v) for v in (temperature, top_k, counter, top_p, repetition_penalty)]
    if top_n is not None:
        vals.append(list(top_n))
    if not all(len(v) == B for v in vals):
        raise VclError(f"temperature / top_k / counter / top_p / repetition_penalty (/ top_n) need {B} entries each")
    if token_sets is not None:
        assert token_sets.is_cuda and token_sets.dtype == torch.int32 and token_sets.is_contiguous()
        assert tuple(token_sets.shape) == (B, token_set_words(ld))
    out = torch.empty(B, dtype=torch.int32, device=logits.device)
    ids = lp = None
    if top_n is not None:
        ids = torch.full((B, LOGPROB_PLACES), -1, dtype=torch.int32, device=logits.device)
        lp = torch.full((B, LOGPROB_PLACES), float("nan"), dtype=torch.float32, device=logits.device)
    ints = lambda v: (c_int32 * B)(*[int(x) for x in v])   # noqa: E731
    flts = lambda v: (c_float * B)(*[float(x) for x in v])   # noqa: E731
    check(lib().vcl_op_sample_ex(c_void_p(logits.data_ptr()), logits.stride(0), B, ld, flts(vals[0]), ints(vals[1]),
                                 _seeds(seed, B), ints(vals[2]), flts(vals[3]), flts(vals[4]), ptr(token_sets),
                                 ints(vals[5]) if top_n is not None else None, ptr(out), ptr(ids), ptr(lp),
                                 cur_stream()))
    return out if top_n is None else (out, ids, lp)


def op_sample_warpers(logits, temperature, top_k, seed, counter, top_p, repetition_penalty, min_p, typical_p,
                      epsilon, eta, token_sets=None, top_n=None):
    """The 32-bit sampler with HF's min-p / typical / epsilon / eta warpers alone (vcl_op_sample_warpers):
    op_sample_ex's arguments plus B host values each of min_p (0: off), typical_p (1: off), epsilon and eta (0: off).
    Returns what op_sample_ex returns."""
    B, ld = logits.shape
    assert logits.dtype == torch.float32 and logits.stride(1) == 1
    vals = [list(v) for v in (temperature, top_k, counter, top_p, repetition_penalty, min_p, typical_p, epsilon, eta)]
    if top_n is not None:
        vals.append(list(top_n))
    if not all(len(v) == B for v in vals):
        raise VclError(f"every per-row setting needs {B} entries")
    if token_sets is not None:
        assert token_sets.is_cuda and token_sets.dtype == torch.int32 and token_sets.is_contiguous()
        assert tuple(token_sets.shape) == (B, token_set_words(ld))
    out = torch.empty(B, dtype=torch.int32, device=logits.device)
    ids = lp = None
    if top_n is not None:
        ids = torch.full((B, LOGPROB_PLACES), -1, dtype=torch.int32, device=logits.device)
        lp = torch.full((B, LOGPROB_PLACES), float("nan"), dtype=torch.float32, device=logits.device)
    ints = lambda v: (c_int32 * B)(*[int(x) for x in v])   # noqa: E731
    flts = lambda v: (c_float * B)(*[float(x) for x in v])   # noqa: E731
    check(lib().vcl_op_sample_warpers(c_void_p(logits.data_ptr()), logits.stride(0), B, ld, flts(vals[0]),
                                      ints(vals[1]), _seeds(seed, B), ints(vals[2]), flts(vals[3]), flts(vals[4]),
                                      ptr(token_sets), flts(vals[5]), flts(vals[6]), flts(vals[7]), flts(vals[8]),
                                      ints(vals[9]) if top_n is not None else None, ptr(out), ptr(ids), ptr(lp),
                                      cur_stream()))
    return out if top_n is None else (out, ids, lp)


BAN_WORDS_MAX = 1024          # include/vcl.h: VCL_BAN_WORDS_MAX, the int32 of one entry's bad-words list


def op_guidance(logits, partner, scale):
    """Classifier-free guidance alone (vcl_op_guidance): logits [B, V] fp32 on the device; partner / scale B host
    values (partner -1: the row is left as it is). Returns a new [B, V] fp32 tensor whose guided rows b hold
    scale[b] * (log_softmax(row b) - log_softmax(row partner[b])) + log_softmax(row partner[b]) by the fp32 rule of
    DESIGN.md section 3."""
    B, V = logits.shape
    assert logits.dtype == torch.float32 and logits.stride(1) == 1
    if len(partner) != B or len(scale) != B:
        raise VclError(f"partner / scale need {B} entries each")
    out = torch.empty_like(logits, memory_format=torch.contiguous_format)
    if logits.stride(0) != V:
        logits = logits.contiguous()
    check(lib().vcl_op_guidance(c_void_p(logits.data_ptr()), V, B, V, (c_int32 * B)(*[int(u) for u in partner]),
                                (c_float * B)(*[float(g) for g in scale]), ptr(out), cur_stream()))
    return out


def ban_words(words):
    """A list of bad words (each a non-empty list of ids) -> the BAN_WORDS_MAX int32 of vcl_llm_set_bans' format:
    records (L, id_0 .. id_{L-1}), then zeros"""
    flat = []
    for w in words:
        flat += [len(w)] + [int(x) for x in w]
    if len(flat) > BAN_WORDS_MAX:
        raise VclError(f"bad words take {len(flat)} int32 (a length and the ids of each word), more than the "
                       f"{BAN_WORDS_MAX} of one entry")
    return flat + [0] * (BAN_WORDS_MAX - len(flat))


def op_sample_bans(logits, temperature, top_k, seed, counter, top_p, repetition_penalty, histories, ngram, eos,
                   eos_from_col, words, token_sets=None, top_n=None):
    """The 32-bit sampler with the ban stage alone (vcl_op_sample_bans): op_sample_ex's arguments plus histories
    [B, hist_ld] int32 on the device (row b draws at column counter[b] < hist_ld, after h[0 .. counter[b]), and writes
    its token there), and per row the n-gram size ngram[b] (0: off), eos[b] (-1: off) with eos_from_col[b], and
    words[b], a list of bad words (lists of ids). Returns what op_sample_ex returns."""
    B, ld = logits.shape
    assert logits.dtype == torch.float32 and logits.stride(1) == 1
    vals = [list(v) for v in (temperature, top_k, counter, top_p, repetition_penalty, ngram, eos, eos_from_col, words)]
    if top_n is not None:
        vals.append(list(top_n))
    if not all(len(v) == B for v in vals):
        raise VclError(f"every per-row setting needs {B} entries")
    assert histories.is_cuda and histories.dtype == torch.int32 and histories.dim() == 2 and histories.shape[0] == B
    assert histories.stride(1) == 1
    if token_sets is not None:
        assert token_sets.is_cuda and token_sets.dtype == torch.int32 and token_sets.is_contiguous()
        assert tuple(token_sets.shape) == (B, token_set_words(ld))
    out = torch.empty(B, dtype=torch.int32, device=logits.device)
    ids = lp = None
    if top_n is not None:
        ids = torch.full((B, LOGPROB_PLACES), -1, dtype=torch.int32, device=logits.device)
        lp = torch.full((B, LOGPROB_PLACES), float("nan"), dtype=torch.float32, device=logits.device)
    ints = lambda v: (c_int32 * len(v))(*[int(x) for x in v])   # noqa: E731
    flts = lambda v: (c_float * B)(*[float(x) for x in v])   # noqa: E731
    flat = [x for w in vals[8] for x in ban_words(w)]
    check(lib().vcl_op_sample_bans(c_void_p(logits.data_ptr()), logits.stride(0), B, ld, flts(vals[0]), ints(vals[1]),
                                   _seeds(seed, B), ints(vals[2]), flts(vals[3]), flts(vals[4]), ptr(token_sets),
                                   ptr(histories), histories.stride(0), ints(vals[5]), ints(vals[6]), ints(vals[7]),
                                   ints(flat), ints(vals[9]) if top_n is not None else None, ptr(out), ptr(ids),
                                   ptr(lp), cur_stream()))
    return out if top_n is None else (out, ids, lp)


BEAM_MAX = 8                  # include/vcl.h: VCL_BEAM_MAX, the most beams per item


def beam_records(rec):
    """records int32 [..., K, 3] (vcl_beam_record: f32 score bits, beam, token) -> (score f32, beam int64, token
    int64), each [..., K]"""
    return rec[..., 0].view(torch.float32), rec[..., 1].to(torch.int64), rec[..., 2].to(torch.int64)


def op_beam_select(logits, scores, num_beams, eos=-1, last_step=False):
    """One beam-search step alone (vcl_op_beam_select): logits [B * k, ld] fp32 on the device (bf16 values), scores
    [B * k] fp32 running scores. Returns (records int32 [B, 2k, 3], picks int32 [B, k]) on the device (beam_records
    unpacks the records)."""
    Bk, ld = logits.shape
    k = int(num_beams)
    assert logits.dtype == torch.float32 and logits.stride(1) == 1 and Bk % k == 0
    sc = scores.to(device=logits.device, dtype=torch.float32).contiguous()
    assert sc.numel() == Bk
    B = Bk // k
    rec = torch.empty(B, 2 * k, 3, dtype=torch.int32, device=logits.device)
    picks = torch.empty(B, k, dtype=torch.int32, device=logits.device)
    check(lib().vcl_op_beam_select(c_void_p(logits.data_ptr()), logits.stride(0), B, k, ld, ptr(sc), int(eos),
                                   int(bool(last_step)), ptr(rec), ptr(picks), cur_stream()))
    return rec, picks


CS_MAX_K = 64                 # include/vcl.h: VCL_CS_MAX_K, the most contrastive-search candidates per prompt


def cs_record_len(k):
    """f32 words per contrastive-search step record (include/vcl.h: VCL_CS_RECORD)"""
    return 2 + 4 * int(k)


def cs_records(rec, k):
    """records f32 [..., 2 + 4k] -> dict of token / pick int64 [...] and cand int64, p, cos, score f32 [..., k]"""
    k = int(k)
    return {"token": rec[..., 0].to(torch.int64), "pick": rec[..., 1].to(torch.int64),
            "cand": rec[..., 2:2 + k].to(torch.int64), "p": rec[..., 2 + k:2 + 2 * k],
            "cos": rec[..., 2 + 2 * k:2 + 3 * k], "score": rec[..., 2 + 3 * k:2 + 4 * k]}


def op_contrastive_rank(ctx, n_pad, n_ctx, hid, p, cand_tok, penalty_alpha):
    """The contrastive rank alone (vcl_op_contrastive_rank): ctx [B, rows, D] bf16 on the device (row n_ctx receives
    each prompt's chosen row), n_pad [B] host ints, hid [B * k, D] bf16, p [B * k] f32, cand_tok [B * k] int32.
    Returns records f32 [B, 2 + 4k] on the device (cs_records unpacks them)."""
    B, rows, D = ctx.shape
    Bk = hid.shape[0]
    assert ctx.dtype == hid.dtype == torch.bfloat16 and ctx.is_contiguous() and hid.is_contiguous() and Bk % B == 0
    k = Bk // B
    pd = p.to(device=ctx.device, dtype=torch.float32).contiguous()
    td = cand_tok.to(device=ctx.device, dtype=torch.int32).contiguous()
    rec = torch.empty(B, cs_record_len(k), dtype=torch.float32, device=ctx.device)
    check(lib().vcl_op_contrastive_rank(c_void_p(ctx.data_ptr()), rows, _host_pads(n_pad, B), int(n_ctx), B, k, D,
                                        ptr(hid), ptr(pd), ptr(td), float(penalty_alpha), ptr(rec), cur_stream()))
    return rec


def op_gemv(x, w, res=None, norm_w=None, eps=0.0):
    B, K = x.shape
    N = w.shape[0]
    out = torch.empty(B, N, dtype=torch.bfloat16, device=x.device)
    check(lib().vcl_op_gemv(ptr(x), ptr(w), ptr(out), ptr(res), ptr(norm_w), eps, B, N, K, cur_stream()))
    return out


def op_gemv_fp8(x, w, res=None, norm_w=None, eps=0.0):
    """op_gemv with w quantized to E4M3 by the load-time quantizer and the fp8 ring kernels (vcl_op_gemv_fp8);
    equals op_gemv(x, W~) bit for bit, W~ = op_quantize_fp8(w)[0]."""
    B, K = x.shape
    N = w.shape[0]
    out = torch.empty(B, N, dtype=torch.bfloat16, device=x.device)
    check(lib().vcl_op_gemv_fp8(ptr(x), ptr(w), ptr(out), ptr(res), ptr(norm_w), eps, B, N, K, cur_stream()))
    return out


GEMV_RES, GEMV_SWIGLU, GEMV_LOGITS = 0, 1, 3   # vcl_op_gemv_ex: the fused epilogues of the decode projections


def gemv_grid(N):
    """CTAs of a 1..4-row decode projection over N rows: the rows of the arg-max partials of vcl_op_gemv_ex"""
    return min((N + 15) // 16, torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count)


def op_gemv_ex(x, w, mode, fp8=False, norm_w=None, eps=0.0, out=None, logits=True, partials=False):
    """One decode projection through a fused epilogue (vcl_op_gemv_ex), x [B, K] bf16, w [N, K] bf16; fp8: the
    E4M3 kernels on the quantized w (equal to the bf16 launch on W~ = op_quantize_fp8(w)[0]).
    RES (no residual): returns out [B, N] bf16. SWIGLU: out [B, N/2] bf16 at B <= 4, the flat xwin buffer at 5..64
    (see xwin_offset; `out` may be given, e.g. pre-filled with a sentinel). LOGITS: returns (logits [B, N] fp32 or
    None, partials int32 [gemv_grid(N), B, 2] or None: the value's bits and the row of each CTA's arg-max)."""
    B, K = x.shape
    N = w.shape[0]
    lg = pt = None
    if mode == GEMV_LOGITS:
        lg = torch.empty(B, N, dtype=torch.float32, device=x.device) if logits else None
        pt = torch.empty(gemv_grid(N), B, 2, dtype=torch.int32, device=x.device) if partials else None
    elif out is None:
        if mode == GEMV_SWIGLU and B > 4:
            out = torch.empty((N // 2 + XWIN_KC - 1) // XWIN_KC * B * XWIN_PITCH, dtype=torch.bfloat16, device=x.device)
        else:
            out = torch.empty(B, N // 2 if mode == GEMV_SWIGLU else N, dtype=torch.bfloat16, device=x.device)
    check(lib().vcl_op_gemv_ex(ptr(x), ptr(w), int(bool(fp8)), mode, ptr(out), None, ptr(lg), ptr(pt), ptr(norm_w),
                               eps, B, N, K, cur_stream()))
    return (lg, pt) if mode == GEMV_LOGITS else out


def tiled_elems(N, K):
    """elements (bytes for fp8) of the slot-ordered decode copy of an [N, K] matrix"""
    return (N + 15) // 16 * 16 * K


def op_quantize_fp8(w):
    """The load-time E4M3 quantizer alone (vcl_op_quantize_fp8), rows in order: w [N, K] bf16 ->
    (W~ [N, K] bf16, codes uint8 [tiled_elems(N, K)] in the decode kernels' slot order, scales [N] fp32 = 2^e)."""
    N, K = w.shape
    deq = torch.empty_like(w)
    codes = torch.empty(tiled_elems(N, K), dtype=torch.uint8, device=w.device)
    scales = torch.empty(N, dtype=torch.float32, device=w.device)
    check(lib().vcl_op_quantize_fp8(ptr(w), N, K, ptr(deq), ptr(codes), ptr(scales), cur_stream()))
    return deq, codes, scales


XWIN_KC, XWIN_PITCH = 512, 544     # kernels.h: the window-major activation layout of the 5..64-clip decode kernels


def xwin_offset(b, k, B):
    """element (b, k) of a [B][K] activation in the xwin layout (kernels.h)"""
    return ((k // XWIN_KC) * B + b) * XWIN_PITCH + k % XWIN_KC


def op_decode_attention(q, k, v, kv_len, n_pad, pos_dev=None, scale=128 ** -0.5, o_xwin=False, table=None,
                        n_blocks=0, blk=0, s_max=None, out=None):
    """The decode attention kernel alone (vcl_op_decode_attention). q [B, q_ld] bf16 (head h at columns
    h*128 ..; q_ld >= H*128), n_pad / pos_dev int32 [B] on the device (pos_dev optional). Contiguous cache (table
    None): k / v [B, H, s_max, 128] bf16. Paged (vcl_op_decode_attention_paged): k / v are one layer's K / V planes of
    block 0 of a pool (any [.., H, 128, 128] views), table [B, ceil(s_max / 128)] host ints, n_blocks blocks blk
    elements apart, s_max the columns a clip may hold. Returns o [B, H*128], or with o_xwin the flat xwin buffer (see
    xwin_offset); out if given."""
    B = q.shape[0]
    H = k.shape[-3]
    assert k.shape[-1] == 128 and q.stride(1) == 1 and v.shape == k.shape
    if out is not None:
        o = out
    elif o_xwin:
        o = torch.empty((H * 128 + XWIN_KC - 1) // XWIN_KC * B * XWIN_PITCH, dtype=torch.bfloat16, device=q.device)
    else:
        o = torch.empty(B, H * 128, dtype=torch.bfloat16, device=q.device)
    if table is None:
        assert k.dim() == 4 and k.shape[0] == B
        check(lib().vcl_op_decode_attention(ptr(q), q.stride(0), ptr(k), ptr(v), ptr(o), B, H, k.shape[2],
                                            int(kv_len), ptr(pos_dev), ptr(n_pad), scale, int(o_xwin), cur_stream()))
    else:
        vals = table.tolist() if hasattr(table, "tolist") else table
        assert len(vals) == B and all(len(r) == (int(s_max) + 127) // 128 for r in vals)
        check(lib().vcl_op_decode_attention_paged(ptr(q), q.stride(0), c_void_p(k.data_ptr()), c_void_p(v.data_ptr()),
                                                  ptr(o), B, H, int(s_max), int(kv_len), ptr(pos_dev), ptr(n_pad),
                                                  scale, int(o_xwin), _ints([b for r in vals for b in r]),
                                                  int(n_blocks), int(blk), cur_stream()))
    return o


def _rows_view(t, what):
    """a [rows, ld] bf16 device tensor with unit column stride -> (pointer, row pitch)"""
    assert t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1, what
    return c_void_p(t.data_ptr()), t.stride(0)


def _ints(vals):
    vals = [int(x) for x in vals]
    return (c_int32 * len(vals))(*vals)


def op_attention_cached(q, k, v, start_pos, n_pad=None, out=None):
    """The prefill attention over the cache alone (vcl_op_attention_cached): q [B*S, q_ld] bf16 (head h at columns
    h*128 ..), k / v [B, H, s_max, 128] bf16 caches, the queries at positions start_pos .. start_pos + S - 1,
    n_pad None or B host ints. Returns o [B*S, H*128] (out if given)."""
    B, H, s_max, hd = k.shape
    assert hd == 128 and v.shape == k.shape and k.is_contiguous() and v.is_contiguous()
    qp, q_ld = _rows_view(q, "q")
    S = q.shape[0] // B
    o = out if out is not None else torch.empty(B * S, H * 128, dtype=torch.bfloat16, device=q.device)
    pads = None if n_pad is None else _host_pads(n_pad, B)
    check(lib().vcl_op_attention_cached(qp, q_ld, ptr(k), ptr(v), ptr(o), B, H, s_max, int(start_pos), S, pads,
                                        cur_stream()))
    return o


def op_attention_packed(q, k, v, slots, starts, lens, flash=None, table=None, n_blocks=0, blk=0, s_max=None,
                        out=None):
    """The packed prefill attention alone (vcl_op_attention_packed): sequence i is lens[i] query rows of q [sum lens,
    q_ld] at positions starts[i] .. of slot slots[i] (host ints), on the flash kernel when flash[i] (paged only).
    Contiguous cache (table None): k / v [n_slots, H, s_max, 128]. Paged: k / v are one layer's K / V planes of block 0
    of a pool (any [.., H, 128, 128] views), table [n_slots, table_row] host ints, n_blocks blocks blk elements apart,
    s_max the columns a slot may hold. Returns o [sum lens, H*128] (out if given)."""
    n = len(slots)
    qp, q_ld = _rows_view(q, "q")
    H = k.shape[-3]
    if table is None:
        n_slots, _, s_max, _ = k.shape
        assert k.is_contiguous() and v.shape == k.shape and v.is_contiguous()
        tab, row = None, 0
    else:
        vals = table.tolist() if hasattr(table, "tolist") else table
        n_slots, row = len(vals), len(vals[0])
        tab = _ints([b for r in vals for b in r])
    o = out if out is not None else torch.empty(sum(int(x) for x in lens), H * 128, dtype=torch.bfloat16,
                                                device=q.device)
    check(lib().vcl_op_attention_packed(qp, q_ld, c_void_p(k.data_ptr()), c_void_p(v.data_ptr()), ptr(o), H,
                                        int(s_max), n_slots, n, _ints(slots), _ints(starts), _ints(lens),
                                        None if flash is None else _ints(flash), tab, row, int(n_blocks), int(blk),
                                        cur_stream()))
    return o


def op_attention_appended(q, k, v, slots, starts, lens, out=None):
    """The attention of candidate scoring alone (vcl_op_attention_appended): op_attention_packed on a contiguous cache
    k / v [n_slots, H, s_max, 128], each sequence on the kernel the contiguous continued prefill takes (flash past 512
    keys). Returns o [sum lens, H*128] (out if given)."""
    n_slots, H, s_max, _ = k.shape
    assert k.is_contiguous() and v.shape == k.shape and v.is_contiguous()
    qp, q_ld = _rows_view(q, "q")
    o = out if out is not None else torch.empty(sum(int(x) for x in lens), H * 128, dtype=torch.bfloat16,
                                                device=q.device)
    check(lib().vcl_op_attention_appended(qp, q_ld, ptr(k), ptr(v), ptr(o), H, int(s_max), n_slots, len(slots),
                                          _ints(slots), _ints(starts), _ints(lens), cur_stream()))
    return o


# ---------------------------------------------------------------------------------------------
# engine handle
# ---------------------------------------------------------------------------------------------
def _tensor_array(state: dict, keep: list):
    """Pack a {name: cuda bf16 tensor} dict into a vcl_tensor array (tensors kept alive in `keep`)."""
    arr = (vcl_tensor * len(state))()
    for i, (name, t) in enumerate(state.items()):
        t = t.detach()
        if t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous():
            t = t.to(device="cuda", dtype=torch.bfloat16).contiguous()
        keep.append(t)
        arr[i].name = name.encode()
        arr[i].data = t.data_ptr()
        arr[i].ndim = t.dim()
        for d in range(t.dim()):
            arr[i].shape[d] = t.shape[d]
    return arr


def _host_pads(n_pad, B: int):
    """n_pad (sequence / tensor of B ints, any device) -> ctypes int32[B] in host memory."""
    vals = n_pad.tolist() if isinstance(n_pad, torch.Tensor) else list(n_pad)
    if len(vals) != B:
        raise VclError(f"n_pad has {len(vals)} entries for {B} rows")
    return (c_int32 * B)(*[int(v) for v in vals])


def launch_count() -> int:
    return int(lib().vcl_launch_count())


class Engine:
    """Owns one vcl_handle (one per process / GPU)."""

    def __init__(self, cfg: vcl_config, kv_blocks: int | None = None):
        """cfg: a vcl_config (or vcl_config_ex). kv_blocks: > 0 makes the KV cache paged (vcl_config.kv_blocks);
        None keeps cfg's own (0 for a plain vcl_config)."""
        ex = vcl_config_ex()
        ctypes.memmove(ctypes.addressof(ex), ctypes.addressof(cfg), ctypes.sizeof(cfg))
        if kv_blocks is not None:
            ex.kv_blocks = int(kv_blocks)
        cfg = self.cfg = ex
        self._h = c_void_p()
        check(lib().vcl_create(ctypes.byref(self._h), ctypes.byref(cfg)))
        g = cfg.image_size // cfg.patch_size
        self.P = g * g
        self.NV = cfg.n_temporal + self.P

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().vcl_destroy(self._h)
            self._h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights ----
    def load_clip(self, state: dict):
        keep: list = []
        arr = _tensor_array(state, keep)
        torch.cuda.synchronize()
        check(lib().vcl_load_clip_weights(self._h, arr, len(state)))

    def load_llm(self, state: dict, weight_format: str = "bf16"):
        """weight_format "bf16" (vcl_load_llm_weights) or "fp8_e4m3" (vcl_load_llm_weights_ex: the streamed
        matrices as E4M3 codes with power-of-two row scales; the engine then computes with the dequantized
        weights W~). Any other value raises ValueError before anything is loaded."""
        fmt = weight_format_code(weight_format)
        keep: list = []
        arr = _tensor_array(state, keep)
        torch.cuda.synchronize()
        if fmt == WEIGHTS_BF16:
            check(lib().vcl_load_llm_weights(self._h, arr, len(state)))
        else:
            check(lib().vcl_load_llm_weights_ex(self._h, arr, len(state), fmt))

    # ---- vision ----
    @staticmethod
    def _pixels(pixels: torch.Tensor):
        """-> (contiguous tensor, format code, frame height, frame width); the layout is told by the
        dtype: uint8 = raw [N,H,W,3] frames, floating = normalised [N,3,H,W] pixel_values."""
        if pixels.dim() != 4:
            raise VclError(f"pixels must be 4-D, got shape {tuple(pixels.shape)}")
        if pixels.dtype == torch.uint8:
            if pixels.shape[3] != 3:
                raise VclError(f"uint8 frames must be [N,H,W,3] (channels last), got {tuple(pixels.shape)}")
            return pixels.contiguous(), PIXELS_U8_NHWC, pixels.shape[1], pixels.shape[2]
        if pixels.shape[1] != 3:
            raise VclError(f"pixel_values must be [N,3,H,W], got {tuple(pixels.shape)}")
        return pixels.to(torch.bfloat16).contiguous(), PIXELS_BF16_NCHW, pixels.shape[2], pixels.shape[3]

    def clip_encode(self, pixels: torch.Tensor, n_layers: int | None = None) -> torch.Tensor:
        """pixels: [N,3,H,W] bf16 (normalised) or [N,H,W,3] uint8 -> hidden_states[n_layers] [N,1+P,C]."""
        pixels, fmt, fh, fw = self._pixels(pixels)
        n = pixels.shape[0]
        nl = self.cfg.clip_layers if n_layers is None else n_layers
        out = torch.empty(n, self.P + 1, self.cfg.clip_hidden, dtype=torch.bfloat16, device=pixels.device)
        check(lib().vcl_clip_encode(self._h, ptr(pixels), fmt, n, fh, fw, nl, ptr(out), cur_stream()))
        return out

    def clip_features(self, pixels: torch.Tensor, out_dtype=torch.float16, out=None) -> torch.Tensor:
        pixels, fmt, fh, fw = self._pixels(pixels)
        if out is None:
            out = torch.empty(self.NV, self.cfg.clip_hidden, dtype=out_dtype, device=pixels.device)
        else:
            out_dtype = out.dtype
            assert out.shape == (self.NV, self.cfg.clip_hidden)
        check(lib().vcl_clip_features(self._h, ptr(pixels), fmt, pixels.shape[0], fh, fw, ptr(out),
                                      _dtype_code(out_dtype), cur_stream()))
        return out

    # ---- language model ----
    def prefill(self, ids, video_feats, vid_start, n_layers=None, want_hidden=False, want_logits=False,
                want_token=True, tok_out=None, n_pad=None):
        """n_pad: None (vcl_llm_prefill), or B left-padding counts (vcl_llm_prefill_padded; the cache stays
        padded for the appends and decode steps that follow)."""
        B, S = ids.shape
        nl = self.cfg.llm_layers if n_layers is None else n_layers
        dev = ids.device
        hidden = torch.empty(B, S, self.cfg.llm_hidden, dtype=torch.bfloat16, device=dev) if want_hidden else None
        logits = torch.empty(B, self.cfg.vocab, dtype=torch.float32, device=dev) if want_logits else None
        tok = tok_out if tok_out is not None else (
            torch.empty(B, dtype=torch.int32, device=dev) if want_token else None)
        vf = None
        if video_feats is not None:
            vf = video_feats.to(torch.bfloat16).contiguous()
            assert vf.shape == (B, self.NV, self.cfg.clip_hidden), vf.shape
        if n_pad is None:
            check(lib().vcl_llm_prefill(self._h, ptr(ids.contiguous()), ptr(vf), ptr(vid_start.contiguous()), B, S,
                                        nl, ptr(hidden), ptr(logits), ptr(tok), cur_stream()))
        else:
            check(lib().vcl_llm_prefill_padded(self._h, ptr(ids.contiguous()), ptr(vf), ptr(vid_start.contiguous()),
                                               _host_pads(n_pad, B), B, S, nl, ptr(hidden), ptr(logits), ptr(tok),
                                               cur_stream()))
        return hidden, logits, tok

    def score(self, ids, video_feats, vid_start, labels=None, n_pad=None, want_logits=False):
        """Full-depth prefill with lm_head at every position (vcl_llm_score). labels [B, S] (-100 ignored; HF's
        shift: column s is scored against labels[:, s+1]). Returns (logits [B,S,vocab] bf16 | None,
        nll [B,S-1] fp32 | None, loss 0-d fp32 | None); nll and loss need labels. n_pad as in prefill."""
        B, S = ids.shape
        dev = ids.device
        logits = torch.empty(B, S, self.cfg.vocab, dtype=torch.bfloat16, device=dev) if want_logits else None
        nll = loss = lab = None
        if labels is not None:
            lab = labels.to(device=dev, dtype=torch.int64).contiguous()
            assert lab.shape == (B, S), lab.shape
            nll = torch.empty(B, S - 1, dtype=torch.float32, device=dev)
            loss = torch.empty((), dtype=torch.float32, device=dev)
        vf = None
        if video_feats is not None:
            vf = video_feats.to(torch.bfloat16).contiguous()
            assert vf.shape == (B, self.NV, self.cfg.clip_hidden), vf.shape
        pads = None if n_pad is None else _host_pads(n_pad, B)
        check(lib().vcl_llm_score(self._h, ptr(ids.contiguous()), ptr(vf), ptr(vid_start.contiguous()), pads, B, S,
                                  ptr(lab), ptr(logits), ptr(nll), ptr(loss), cur_stream()))
        return logits, nll, loss

    def prefill_states(self, ids, video_feats, vid_start, want_logits=False):
        """Full-depth prefill keeping every hidden state: ([L+1, B, S, D] bf16 raw layer outputs,
        last-position logits [B, vocab] | None)."""
        B, S = ids.shape
        dev = ids.device
        states = torch.empty(self.cfg.llm_layers + 1, B, S, self.cfg.llm_hidden, dtype=torch.bfloat16, device=dev)
        logits = torch.empty(B, self.cfg.vocab, dtype=torch.float32, device=dev) if want_logits else None
        vf = None
        if video_feats is not None:
            vf = video_feats.to(torch.bfloat16).contiguous()
            assert vf.shape == (B, self.NV, self.cfg.clip_hidden), vf.shape
        check(lib().vcl_llm_prefill_states(self._h, ptr(ids.contiguous()), ptr(vf), ptr(vid_start.contiguous()), B, S,
                                           ptr(states), ptr(logits), cur_stream()))
        return states, logits

    def prefill_append(self, ids, start_pos, want_hidden=False, want_logits=False, want_token=True):
        """Continue the cached sequences with `ids` [B, S] (text only) at positions start_pos.. ;
        returns (hidden [B,S,D] | None, logits [B,vocab] | None, next token [B] | None)."""
        B, S = ids.shape
        dev = ids.device
        hidden = torch.empty(B, S, self.cfg.llm_hidden, dtype=torch.bfloat16, device=dev) if want_hidden else None
        logits = torch.empty(B, self.cfg.vocab, dtype=torch.float32, device=dev) if want_logits else None
        tok = torch.empty(B, dtype=torch.int32, device=dev) if want_token else None
        check(lib().vcl_llm_prefill_append(self._h, ptr(ids.contiguous()), B, S, int(start_pos), ptr(hidden),
                                           ptr(logits), ptr(tok), cur_stream()))
        return hidden, logits, tok

    def decode_step(self, tok_in, pos, want_logits=False):
        B = tok_in.shape[0]
        logits = torch.empty(B, self.cfg.vocab, dtype=torch.float32, device=tok_in.device) if want_logits else None
        tok = torch.empty(B, dtype=torch.int32, device=tok_in.device)
        check(lib().vcl_llm_decode_step(self._h, ptr(tok_in.contiguous()), B, pos, ptr(logits), ptr(tok),
                                        cur_stream()))
        return logits, tok

    def decode_loop(self, first_tok, S, n_new, out=None):
        B = first_tok.shape[0]
        if out is None:
            out = torch.empty(B, n_new, dtype=torch.int32, device=first_tok.device)
        check(lib().vcl_llm_decode_loop(self._h, ptr(first_tok.contiguous()), B, S, n_new, ptr(out), cur_stream()))
        return out

    def generate(self, ids, video_feats, vid_start, n_new, n_pad=None):
        """n_pad: None (vcl_llm_generate), or B left-padding counts (vcl_llm_generate_padded)."""
        B, S = ids.shape
        out = torch.empty(B, n_new, dtype=torch.int32, device=ids.device)
        vf = None
        if video_feats is not None:
            vf = video_feats.to(torch.bfloat16).contiguous()
        if n_pad is None:
            check(lib().vcl_llm_generate(self._h, ptr(ids.contiguous()), ptr(vf), ptr(vid_start.contiguous()), B, S,
                                         n_new, ptr(out), cur_stream()))
        else:
            check(lib().vcl_llm_generate_padded(self._h, ptr(ids.contiguous()), ptr(vf), ptr(vid_start.contiguous()),
                                                _host_pads(n_pad, B), B, S, n_new, ptr(out), cur_stream()))
        return out

    # ---- sampling ----
    def set_sampling(self, clips, temperature, top_k, seed):
        """Entries `clips` of the sampling table (vcl_llm_set_sampling): clip / slot clips[i] samples with
        temperature[i] (0: greedy), top_k[i] (0: all tokens) and the 64-bit seed[i]. Host lists of equal length."""
        n = len(clips)
        if not (len(temperature) == len(top_k) == n):
            raise VclError(f"{n} clips, {len(temperature)} temperatures, {len(top_k)} top_k")
        check(lib().vcl_llm_set_sampling(self._h, n, (c_int32 * n)(*[int(b) for b in clips]),
                                         (c_float * n)(*[float(t) for t in temperature]),
                                         (c_int32 * n)(*[int(k) for k in top_k]), _seeds(seed, n), cur_stream()))

    def set_sampling_ex(self, clips, temperature, top_k, seed, top_p, repetition_penalty):
        """set_sampling plus top_p[i] (0 .. 1, 1: off) and repetition_penalty[i] (> 0, 1: off) per entry
        (vcl_llm_set_sampling_ex). Host lists of equal length."""
        n = len(clips)
        if not (len(temperature) == len(top_k) == len(top_p) == len(repetition_penalty) == n):
            raise VclError(f"{n} clips, {len(temperature)} temperatures, {len(top_k)} top_k, {len(top_p)} top_p, "
                           f"{len(repetition_penalty)} repetition_penalty")
        flts = lambda v: (c_float * n)(*[float(x) for x in v])   # noqa: E731
        check(lib().vcl_llm_set_sampling_ex(self._h, n, (c_int32 * n)(*[int(b) for b in clips]), flts(temperature),
                                            (c_int32 * n)(*[int(k) for k in top_k]), _seeds(seed, n), flts(top_p),
                                            flts(repetition_penalty), cur_stream()))

    def set_warpers(self, clips, min_p, typical_p, epsilon, eta):
        """HF's min-p / typical / epsilon / eta warpers of entries `clips` (vcl_llm_set_warpers): min_p[i] (0: off),
        typical_p[i] (1: off), epsilon[i] and eta[i] (0: off). set_sampling / set_sampling_ex turn them off for the
        entries they write, so call this after them. Host lists of equal length."""
        n = len(clips)
        if not (len(min_p) == len(typical_p) == len(epsilon) == len(eta) == n):
            raise VclError(f"{n} clips, {len(min_p)} min_p, {len(typical_p)} typical_p, {len(epsilon)} epsilon, "
                           f"{len(eta)} eta")
        flts = lambda v: (c_float * n)(*[float(x) for x in v])   # noqa: E731
        check(lib().vcl_llm_set_warpers(self._h, n, (c_int32 * n)(*[int(b) for b in clips]), flts(min_p),
                                        flts(typical_p), flts(epsilon), flts(eta), cur_stream()))

    def set_token_set(self, entry, ids):
        """Entry `entry`'s token set of the repetition penalty becomes the ids of `ids` (any int tensor or list;
        vcl_llm_set_token_set)"""
        t = torch.as_tensor(ids).reshape(-1).to(device="cuda", dtype=torch.int64).contiguous()
        check(lib().vcl_llm_set_token_set(self._h, int(entry), ptr(t) if t.numel() else None, t.numel(), cur_stream()))

    def read_token_set(self, entry):
        """Entry `entry`'s token set (vcl_llm_read_token_set) as a sorted int64 tensor of token ids on the host"""
        words = token_set_words(self.cfg.vocab)
        bits = torch.empty(words, dtype=torch.int32, device="cuda")
        check(lib().vcl_llm_read_token_set(self._h, int(entry), c_void_p(bits.data_ptr()), cur_stream()))
        b = bits.cpu().to(torch.int64) & 0xFFFFFFFF
        on = ((b[:, None] >> torch.arange(32)) & 1).reshape(-1)
        return on.nonzero()[:, 0]

    # ---- banned tokens ----
    def set_bans(self, clips, ngram, eos, eos_from_col, words):
        """Entries `clips` of the ban table (vcl_llm_set_bans): clip / slot clips[i] bans by the n-gram size ngram[i]
        (0: off), EOS eos[i] (-1: off) before column eos_from_col[i], and the bad words words[i] (a list of lists of
        ids). Host lists of equal length."""
        n = len(clips)
        if not (len(ngram) == len(eos) == len(eos_from_col) == len(words) == n):
            raise VclError(f"{n} clips, {len(ngram)} ngram, {len(eos)} eos, {len(eos_from_col)} eos_from_col, "
                           f"{len(words)} words")
        ints = lambda v: (c_int32 * len(v))(*[int(x) for x in v])   # noqa: E731
        flat = [x for w in words for x in ban_words(w)]
        check(lib().vcl_llm_set_bans(self._h, n, ints(clips), ints(ngram), ints(eos), ints(eos_from_col), ints(flat),
                                     cur_stream()))

    def set_token_history(self, entry, ids):
        """Entry `entry`'s token history, columns 0 .. len(ids) - 1, becomes `ids` (any int tensor or list;
        vcl_llm_set_token_history)"""
        t = torch.as_tensor(ids).reshape(-1).to(device="cuda", dtype=torch.int64).contiguous()
        check(lib().vcl_llm_set_token_history(self._h, int(entry), ptr(t) if t.numel() else None, t.numel(),
                                              cur_stream()))

    def read_token_history(self, entry, first_col, count):
        """Columns first_col .. first_col + count - 1 of entry `entry`'s token history (vcl_llm_read_token_history)
        as an int64 tensor on the host"""
        out = torch.empty(count, dtype=torch.int32, device="cuda")
        check(lib().vcl_llm_read_token_history(self._h, int(entry), int(first_col), int(count),
                                               c_void_p(out.data_ptr()), cur_stream()))
        return out.cpu().to(torch.int64)

    # ---- log-probs of generated tokens ----
    sample_logprobs_op = staticmethod(op_sample_logprobs)

    def set_logprobs(self, clips, top_n):
        """Entries `clips` of the sampling table report log-probs (vcl_llm_set_logprobs): top_n[i] -1 (off), 0 (the
        chosen token) or 1 .. LOGPROBS_MAX alternatives as well. Host lists of equal length."""
        n = len(clips)
        if len(top_n) != n:
            raise VclError(f"{n} clips, {len(top_n)} top_n")
        check(lib().vcl_llm_set_logprobs(self._h, n, (c_int32 * n)(*[int(b) for b in clips]),
                                         (c_int32 * n)(*[int(k) for k in top_n]), cur_stream()))

    # ---- classifier-free guidance ----
    def set_guidance(self, clips, partner, scale):
        """Entries `clips` of the guidance table (vcl_llm_set_guidance): clip clips[i] is guided by the unconditional
        clip partner[i] (-1: off) with scale[i]. Host lists of equal length."""
        n = len(clips)
        if not (len(partner) == len(scale) == n):
            raise VclError(f"{n} clips, {len(partner)} partners, {len(scale)} scales")
        check(lib().vcl_llm_set_guidance(self._h, n, (c_int32 * n)(*[int(b) for b in clips]),
                                         (c_int32 * n)(*[int(u) for u in partner]),
                                         (c_float * n)(*[float(g) for g in scale]), cur_stream()))

    def read_logprobs(self, entry, first_pos, count, ids_out=None, lp_out=None):
        """The log-prob rows of positions first_pos .. first_pos + count - 1 of entry `entry` (vcl_llm_read_logprobs):
        (ids [count, LOGPROB_PLACES] int32, lp [count, LOGPROB_PLACES] f32), device tensors unless given (any
        contiguous device or host tensors of that size)."""
        if ids_out is None:
            ids_out = torch.empty(int(count), LOGPROB_PLACES, dtype=torch.int32, device="cuda")
        if lp_out is None:
            lp_out = torch.empty(int(count), LOGPROB_PLACES, dtype=torch.float32, device="cuda")
        for t, dt in ((ids_out, torch.int32), (lp_out, torch.float32)):
            assert t.dtype == dt and t.is_contiguous() and t.numel() == int(count) * LOGPROB_PLACES
        check(lib().vcl_llm_read_logprobs(self._h, int(entry), int(first_pos), int(count), c_void_p(ids_out.data_ptr()),
                                          c_void_p(lp_out.data_ptr()), cur_stream()))
        return ids_out, lp_out

    # ---- beam search ----
    def beam_start(self, ids, video_feats, vid_start, num_beams, n_new, eos=-1, n_pad=None):
        """Prefill the B prompts once and run beam step 0 (vcl_llm_beam_start): num_beams beams per prompt, n_new
        steps in all, eos -1 for none, n_pad as in prefill. Returns (records int32 [1, B, 2k, 3], picks int32
        [1, B, k]) on the device."""
        B, S = ids.shape
        k = int(num_beams)
        rec = torch.empty(1, B, 2 * k, 3, dtype=torch.int32, device=ids.device)
        picks = torch.empty(1, B, k, dtype=torch.int32, device=ids.device)
        vf = None
        if video_feats is not None:
            vf = video_feats.to(torch.bfloat16).contiguous()
            assert vf.shape == (B, self.NV, self.cfg.clip_hidden), vf.shape
        pads = None if n_pad is None else _host_pads(n_pad, B)
        check(lib().vcl_llm_beam_start(self._h, ptr(ids.contiguous()), ptr(vf), ptr(vid_start.contiguous()), pads, B, S,
                                       k, int(n_new), int(eos), ptr(rec), ptr(picks), cur_stream()))
        self._beam_shape = (B, k)
        return rec, picks

    def beam_decode(self, n_steps):
        """The next n_steps steps of the running beam search (vcl_llm_beam_decode): (records int32 [n, B, 2k, 3],
        picks int32 [n, B, k]) on the device."""
        B, k = self._beam_shape
        rec = torch.empty(int(n_steps), B, 2 * k, 3, dtype=torch.int32, device="cuda")
        picks = torch.empty(int(n_steps), B, k, dtype=torch.int32, device="cuda")
        check(lib().vcl_llm_beam_decode(self._h, int(n_steps), ptr(rec), ptr(picks), cur_stream()))
        return rec, picks

    # ---- contrastive search ----
    def contrastive_start(self, ids, video_feats, vid_start, top_k, penalty_alpha, n_new, n_pad=None):
        """Prefill the B prompts once and run contrastive step 0 (vcl_llm_contrastive_start): top_k candidates per
        prompt, n_new steps in all, n_pad as in prefill. Returns (tokens int32 [1, B], records f32 [1, B, 2 + 4k]) on
        the device (cs_records unpacks them)."""
        B, S = ids.shape
        k = int(top_k)
        tok = torch.empty(1, B, dtype=torch.int32, device=ids.device)
        rec = torch.empty(1, B, cs_record_len(k), dtype=torch.float32, device=ids.device)
        vf = None
        if video_feats is not None:
            vf = video_feats.to(torch.bfloat16).contiguous()
            assert vf.shape == (B, self.NV, self.cfg.clip_hidden), vf.shape
        pads = None if n_pad is None else _host_pads(n_pad, B)
        check(lib().vcl_llm_contrastive_start(self._h, ptr(ids.contiguous()), ptr(vf), ptr(vid_start.contiguous()), pads,
                                              B, S, k, float(penalty_alpha), int(n_new), ptr(tok), ptr(rec),
                                              cur_stream()))
        self._cs_shape = (B, k)
        return tok, rec

    def contrastive_decode(self, n_steps):
        """The next n_steps steps of the running contrastive search (vcl_llm_contrastive_decode): (tokens int32
        [n, B], records f32 [n, B, 2 + 4k]) on the device."""
        B, k = self._cs_shape
        tok = torch.empty(int(n_steps), B, dtype=torch.int32, device="cuda")
        rec = torch.empty(int(n_steps), B, cs_record_len(k), dtype=torch.float32, device="cuda")
        check(lib().vcl_llm_contrastive_decode(self._h, int(n_steps), ptr(tok), ptr(rec), cur_stream()))
        return tok, rec

    # ---- KV cache read-back (tests) ----
    def _cache_shape(self):
        c = self.cfg
        return (c.max_batch, c.llm_heads, c.max_seq, 128)

    def kv_cache(self, layer):
        """(k, v) copies of decoder layer `layer`'s cache, each [max_batch, heads, max_seq, 128] bf16."""
        k = torch.empty(self._cache_shape(), dtype=torch.bfloat16, device="cuda")
        v = torch.empty_like(k)
        check(lib().vcl_kv_cache_copy(self._h, int(layer), 0, ptr(k), ptr(v), cur_stream()))
        return k, v

    def set_kv_cache(self, layer, k, v):
        """Overwrite decoder layer `layer`'s whole cache with k / v ([max_batch, heads, max_seq, 128] bf16)."""
        shape = self._cache_shape()
        assert tuple(k.shape) == shape and tuple(v.shape) == shape and k.dtype == v.dtype == torch.bfloat16
        check(lib().vcl_kv_cache_copy(self._h, int(layer), 1, ptr(k), ptr(v), cur_stream()))

    # ---- paged KV cache (cfg.kv_blocks > 0) ----
    @property
    def kv_blocks(self) -> int:
        return int(self.cfg.kv_blocks)

    @property
    def n_slots(self) -> int:
        """The engine's cache slots (vcl_config.max_slots, 0 meaning min(max_batch, 16))"""
        return int(self.cfg.max_slots) or min(int(self.cfg.max_batch), 16)

    @property
    def table_row(self) -> int:
        """Blocks per slot in the block table: ceil(max_seq / 128)"""
        return (int(self.cfg.max_seq) + KV_BLOCK_COLS - 1) // KV_BLOCK_COLS

    @property
    def block_bytes(self) -> int:
        return kv_block_bytes(self.cfg.llm_layers, self.cfg.llm_heads)

    def block_shape(self):
        """A block as a tensor shape: [layers, 2 (K, V), heads, 128 columns, 128 dims] bf16"""
        c = self.cfg
        return (c.llm_layers, 2, c.llm_heads, KV_BLOCK_COLS, 128)

    def set_block_table(self, table):
        """Write the whole block table (vcl_llm_set_block_table): n_slots rows of table_row block indices (nested
        lists, a numpy array or a tensor on any device). Column c of slot s then lives in block table[s][c // 128]."""
        vals = table.tolist() if hasattr(table, "tolist") else table
        flat = [int(b) for row in vals for b in row]
        if len(vals) != self.n_slots or len(flat) != self.n_slots * self.table_row:
            raise VclError(f"the block table is [{self.n_slots}][{self.table_row}]")
        n = len(flat)
        check(lib().vcl_llm_set_block_table(self._h, (c_int32 * n)(*flat), cur_stream()))

    def swap_buffer(self):
        """A pinned host buffer for one block (kv_block_copy), [block_shape()] bf16"""
        return torch.empty(self.block_shape(), dtype=torch.bfloat16, pin_memory=True)

    def kv_block_copy(self, block, buf, write=False):
        """Copy block `block` whole into buf (write=False) or from buf into the pool (vcl_kv_block_copy). buf: a
        contiguous CUDA tensor or pinned host tensor of block_bytes bytes (e.g. torch.empty(block_shape(), bf16))."""
        assert buf.is_contiguous() and buf.numel() * buf.element_size() == self.block_bytes
        assert buf.is_cuda or buf.is_pinned(), "the block buffer must be device memory or pinned host memory"
        check(lib().vcl_kv_block_copy(self._h, int(block), int(bool(write)), c_void_p(buf.data_ptr()), cur_stream()))
        return buf

    # ---- cache slots (in-flight batching) ----
    def slot_prefill(self, slot, ids, video_feats, vid_start, tok_out=None):
        """One prompt ids [1, S] (or [S]) into cache slot `slot` (vcl_llm_slot_prefill); video_feats [NV, C] /
        [1, NV, C] or None, vid_start [1] int32. Returns its first token, [1] int32 on the device (tok_out if
        given)."""
        ids = ids.reshape(1, -1).contiguous()
        tok = tok_out if tok_out is not None else torch.empty(1, dtype=torch.int32, device=ids.device)
        vf = None
        if video_feats is not None:
            vf = video_feats.to(torch.bfloat16).reshape(1, *video_feats.shape[-2:]).contiguous()
            assert vf.shape == (1, self.NV, self.cfg.clip_hidden), vf.shape
        check(lib().vcl_llm_slot_prefill(self._h, int(slot), ptr(ids), ptr(vf), ptr(vid_start.contiguous()),
                                         ids.shape[1], ptr(tok), cur_stream()))
        return tok

    def slots_prefill(self, slots, ids_list, feats_list, vid_starts, tok_out=None):
        """Prompt i (ids_list[i], [S_i] or [1, S_i]) into cache slot slots[i], all in one packed prefill
        (vcl_llm_slots_prefill). feats_list[i]: its video features [NV, C] / [1, NV, C] or None (text only; its
        vid_starts entry is then ignored), vid_starts: ints. Returns the first tokens, [n] int32 on the device
        (tok_out if given); each equals slot_prefill of that prompt alone, and so does the slot's cache."""
        n = len(slots)
        if not (len(ids_list) == len(feats_list) == len(vid_starts) == n):
            raise VclError(f"{n} slots, {len(ids_list)} prompts, {len(feats_list)} features, {len(vid_starts)} vid_starts")
        ids, lens, packed, vf, vs, tok = self._packed_args(ids_list, feats_list, vid_starts, tok_out)
        check(lib().vcl_llm_slots_prefill(self._h, n, (c_int32 * n)(*[int(s) for s in slots]), (c_int32 * n)(*lens),
                                          ptr(packed), ptr(vf), ptr(vs), ptr(tok), cur_stream()))
        return tok

    def _packed_args(self, ids_list, feats_list, vid_starts, tok_out):
        n, dev = len(ids_list), "cuda"
        ids = [torch.as_tensor(t).reshape(-1) for t in ids_list]
        lens = [t.numel() for t in ids]
        packed = torch.cat([t.to(dev, torch.int64) for t in ids]) if n else torch.empty(0, dtype=torch.int64, device=dev)
        vf = None
        if any(f is not None for f in feats_list):
            vf = torch.zeros(n, self.NV, self.cfg.clip_hidden, dtype=torch.bfloat16, device=dev)
            for i, f in enumerate(feats_list):
                if f is not None:
                    vf[i] = f.reshape(self.NV, self.cfg.clip_hidden)
        vs = torch.tensor([int(v) if f is not None else NO_VIDEO for v, f in zip(vid_starts, feats_list)],
                          dtype=torch.int32, device=dev)
        tok = tok_out if tok_out is not None else torch.empty(n, dtype=torch.int32, device=dev)
        return ids, lens, packed, vf, vs, tok

    def slots_prefill_chunk(self, slots, starts, totals, ids_list, feats_list, vid_starts, tok_out=None):
        """Chunks of prompts into the cache slots of a paged engine, all in one packed pass
        (vcl_llm_slots_prefill_chunk): ids_list[i] ([len_i] or [1, len_i]) is rows starts[i] .. starts[i] + len_i - 1
        of a prompt of totals[i] tokens in slot slots[i], whose earlier rows the slot already holds. feats_list[i] /
        vid_starts[i]: the whole prompt's video features and span start (counted from its first token), as in
        slots_prefill. Returns the token at each chunk's last row, [n] int32 on the device; after a prompt's last
        chunk its slot and that token equal slot_prefill of the whole prompt on a contiguous engine."""
        n = len(slots)
        if not (len(starts) == len(totals) == len(ids_list) == len(feats_list) == len(vid_starts) == n):
            raise VclError(f"{n} slots, {len(starts)} starts, {len(totals)} totals, {len(ids_list)} chunks, "
                           f"{len(feats_list)} features, {len(vid_starts)} vid_starts")
        ids, lens, packed, vf, vs, tok = self._packed_args(ids_list, feats_list, vid_starts, tok_out)
        arr = lambda v: (c_int32 * n)(*[int(x) for x in v])   # noqa: E731
        check(lib().vcl_llm_slots_prefill_chunk(self._h, n, arr(slots), arr(starts), arr(lens), arr(totals),
                                                ptr(packed), ptr(vf), ptr(vs), ptr(tok), cur_stream()))
        return tok

    def slots_prefill_append(self, slots, starts, ids_list, tok_out=None):
        """Text tails appended to the cached sequences of a paged engine's slots, all in one packed pass
        (vcl_llm_slots_prefill_append): ids_list[i] ([len_i] or [1, len_i]) takes positions starts[i] .. of slot
        slots[i], whose columns 0 .. starts[i] - 1 the slot already holds. Returns the token after each tail, [n] int32
        on the device (tok_out if given); it and the slot's new columns equal prefill_append of that tail on a
        contiguous engine holding the same columns."""
        n = len(slots)
        if not (len(starts) == len(ids_list) == n):
            raise VclError(f"{n} slots, {len(starts)} starts, {len(ids_list)} tails")
        ids, lens, packed, _, _, tok = self._packed_args(ids_list, [None] * n, [0] * n, tok_out)
        arr = lambda v: (c_int32 * n)(*[int(x) for x in v])   # noqa: E731
        check(lib().vcl_llm_slots_prefill_append(self._h, n, arr(slots), arr(starts), arr(lens), ptr(packed), ptr(tok),
                                                 cur_stream()))
        return tok

    def slots_fork(self, src, dst, cols):
        """Copy columns 0 .. cols[i] - 1 of cache slot src[i] into slot dst[i], every layer, K and V (vcl_llm_slots_fork;
        contiguous cache). Host lists of equal length."""
        n = len(src)
        if not (len(dst) == len(cols) == n):
            raise VclError(f"{n} sources, {len(dst)} destinations, {len(cols)} column counts")
        arr = lambda v: (c_int32 * max(n, 1))(*[int(x) for x in v])   # noqa: E731
        check(lib().vcl_llm_slots_fork(self._h, n, arr(src), arr(dst), arr(cols), cur_stream()))

    def slots_score_append(self, slots, starts, ids_list, labels_list, lp_out=None, greedy_out=None):
        """Continue slot slots[i]'s cached columns 0 .. starts[i] - 1 with ids_list[i] ([len_i]) and score row t of it
        against labels_list[i][t], all in one packed pass (vcl_llm_slots_score_append; contiguous cache). Returns
        (lp [sum len_i] fp32, greedy [sum len_i] uint8) on the device, sequence i's rows after sequence i - 1's."""
        n = len(slots)
        if not (len(starts) == len(ids_list) == len(labels_list) == n):
            raise VclError(f"{n} slots, {len(starts)} starts, {len(ids_list)} sequences, {len(labels_list)} labels")
        ids, lens, packed, _, _, _ = self._packed_args(ids_list, [None] * n, [0] * n, None)
        lab = torch.cat([torch.as_tensor(t).reshape(-1).to("cuda", torch.int64) for t in labels_list])
        if lab.numel() != packed.numel():
            raise VclError(f"{lab.numel()} labels for {packed.numel()} rows")
        M = packed.numel()
        lp = lp_out if lp_out is not None else torch.empty(M, dtype=torch.float32, device="cuda")
        greedy = greedy_out if greedy_out is not None else torch.empty(M, dtype=torch.uint8, device="cuda")
        arr = lambda v: (c_int32 * n)(*[int(x) for x in v])   # noqa: E731
        check(lib().vcl_llm_slots_score_append(self._h, n, arr(slots), arr(starts), arr(lens), ptr(packed), ptr(lab),
                                               ptr(lp), ptr(greedy), cur_stream()))
        return lp, greedy

    def slot_decode(self, first_tok, positions, n_new, out=None):
        """Slot b is fed first_tok[b] (device int32 [n_slots]) at positions[b] (host ints: the tokens its cache
        holds) and runs n_new-1 greedy steps (vcl_llm_slot_decode); returns [n_slots, n_new] int32, first token
        included."""
        n = first_tok.shape[0]
        pos = list(positions)
        if len(pos) != n:
            raise VclError(f"{len(pos)} positions for {n} slots")
        if out is None:
            out = torch.empty(n, n_new, dtype=torch.int32, device=first_tok.device)
        check(lib().vcl_llm_slot_decode(self._h, ptr(first_tok.contiguous()), (c_int32 * n)(*[int(p) for p in pos]), n,
                                        n_new, ptr(out), cur_stream()))
        return out

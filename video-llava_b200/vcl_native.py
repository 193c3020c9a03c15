"""ctypes binding of libvcl.so (include/vcl.h). PyTorch is used only as the owner of device
memory and streams: every call passes raw device pointers and the current CUDA stream.

There is no fallback: if the shared library is missing or the device is not an sm_90 (H100) GPU the
calls raise.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_uint64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvcl.so")

DTYPE_F16, DTYPE_BF16 = 0, 1
PIXELS_BF16_NCHW, PIXELS_U8_NHWC = 0, 1
PROJ_LINEAR, PROJ_MLP2X_GELU = 0, 1
NO_VIDEO = -2 ** 31          # vid_start value of a text-only row (VCL_NO_VIDEO)
ACT_NONE, ACT_QGELU, ACT_GELU, ACT_SWIGLU = 0, 1, 2, 3


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
    ]


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
    "vcl_clip_encode": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "vcl_st_pool": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                            c_int, c_void_p]),
    "vcl_clip_features": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
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
    "vcl_llm_slot_decode": (c_int, [c_void_p, c_void_p, POINTER(c_int32), c_int, c_int, c_void_p, c_void_p]),
    "vcl_llm_set_sampling": (c_int, [c_void_p, c_int, POINTER(c_int32), POINTER(c_float), POINTER(c_int32),
                                     POINTER(c_uint64), c_void_p]),
    "vcl_launch_count": (ctypes.c_longlong, []),
    "vcl_kv_cache_copy": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_op_decode_attention": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                        c_void_p, c_void_p, c_float, c_int, c_void_p]),
    "vcl_op_cross_entropy": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "vcl_op_gemm": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p,
                            c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "vcl_op_gemm_ex": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p,
                               c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "vcl_op_sample": (c_int, [c_void_p, c_int64, c_int, c_int, POINTER(c_float), POINTER(c_int32), POINTER(c_uint64),
                              POINTER(c_int32), c_void_p, c_void_p]),
    "vcl_op_layernorm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "vcl_op_rmsnorm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "vcl_op_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                 c_float, c_int, c_void_p]),
    "vcl_op_attention_vit": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "vcl_op_gemv": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int,
                            c_int, c_void_p]),
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


def op_attention_vit(qkv, n_frames, S, H):
    """qkv: [n_frames*S, 3*H*64] bf16 -> [n_frames*S, H*64] (ViT attention)."""
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


def op_gemv(x, w, res=None, norm_w=None, eps=0.0):
    B, K = x.shape
    N = w.shape[0]
    out = torch.empty(B, N, dtype=torch.bfloat16, device=x.device)
    check(lib().vcl_op_gemv(ptr(x), ptr(w), ptr(out), ptr(res), ptr(norm_w), eps, B, N, K, cur_stream()))
    return out


XWIN_KC, XWIN_PITCH = 512, 544     # kernels.h: the window-major activation layout of the 5..16-clip decode kernels


def xwin_offset(b, k, B):
    """element (b, k) of a [B][K] activation in the xwin layout (kernels.h)"""
    return ((k // XWIN_KC) * B + b) * XWIN_PITCH + k % XWIN_KC


def op_decode_attention(q, k, v, kv_len, n_pad, pos_dev=None, scale=128 ** -0.5, o_xwin=False):
    """The decode attention kernel alone (vcl_op_decode_attention). q [B, q_ld] bf16 (head h at columns
    h*128 ..; q_ld >= H*128), k / v [B, H, s_max, 128] bf16 caches, n_pad / pos_dev int32 [B] on the device
    (pos_dev optional). Returns o [B, H*128], or with o_xwin the flat xwin buffer (see xwin_offset)."""
    B, H, s_max, hd = k.shape
    assert hd == 128 and q.shape[0] == B and q.stride(1) == 1 and v.shape == k.shape
    if o_xwin:
        o = torch.empty((H * 128 + XWIN_KC - 1) // XWIN_KC * B * XWIN_PITCH, dtype=torch.bfloat16, device=q.device)
    else:
        o = torch.empty(B, H * 128, dtype=torch.bfloat16, device=q.device)
    check(lib().vcl_op_decode_attention(ptr(q), q.stride(0), ptr(k), ptr(v), ptr(o), B, H, s_max, int(kv_len),
                                        ptr(pos_dev), ptr(n_pad), scale, int(o_xwin), cur_stream()))
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

    def __init__(self, cfg: vcl_config):
        self.cfg = cfg
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

    def load_llm(self, state: dict):
        keep: list = []
        arr = _tensor_array(state, keep)
        torch.cuda.synchronize()
        check(lib().vcl_load_llm_weights(self._h, arr, len(state)))

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
        dev = "cuda"
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
        check(lib().vcl_llm_slots_prefill(self._h, n, (c_int32 * n)(*[int(s) for s in slots]), (c_int32 * n)(*lens),
                                          ptr(packed), ptr(vf), ptr(vs), ptr(tok), cur_stream()))
        return tok

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

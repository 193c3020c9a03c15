"""Drop-in for the reference's multimodal model classes on the inference path
(reference: video_chatgpt/model/video_chatgpt.py:16-325 and the bare HF CLIPVisionModel the
reference uses as its vision tower, video_chatgpt/eval/model_utils.py:134-136).

    VisionConfig, VideoChatGPTConfig            :16-34
    VideoChatGPTLlamaModel                      :37-175   (embed + mm_projector + splice + LLaMA stack)
    VideoChatGPTLlamaForCausalLM                :178-321  (forward, generate, prepare_inputs_for_generation)
    CLIPVisionTower                             HF calling convention tower(x, output_hidden_states=True)

All device work goes through one libvcl handle (vcl_native.Engine) shared by the tower and the
language model; these classes only keep state_dicts until the first call, validate inputs the way
the reference does (same ValueError texts for malformed video spans) and translate call
conventions. Differences from the reference, all documented where they occur:
  * compute dtype is bf16 (BASELINE.json); `.half()` is accepted and ignored;
  * `forward` returns logits for the LAST position only, shape [B,1,V] (the reference materialises
    [B,S,V] and every caller on this path reads [:, -1]), unless it is given `labels` (then, as the
    reference, the loss and [B,S,V]) or `logits_to_keep=0` ([B,S,V]). With labels, a right-padded mask
    (train.py's collator) is accepted as well as a left-padded one (score_padding below);
  * the vision tower's `hidden_states` are lazy: an entry is computed when indexed (the path reads [-2]);
    the language model's `hidden_states` are the L+1 tensors HF returns (the last one after the final
    RMSNorm), produced by ONE prefill pass;
  * a batch of prompts of different lengths is LEFT-padded (tokenizer.padding_side = "left") and passed
    with its `attention_mask`, as for HF's LLaMA: every row is computed as if it ran alone (its real tokens
    take positions 0..len-1 and never attend to a pad token). The reference reads the mask but drops the
    positions HF derives from it, and its callers run one video at a time. Right padding and masks with
    holes are rejected (left_padding below).
"""
from __future__ import annotations

import collections
import contextlib
import json
import math
import os
import sys
from types import SimpleNamespace

import torch

_PKG = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)
import vcl_native as vn  # noqa: E402

from ..constants import (DEFAULT_VID_END_TOKEN, DEFAULT_VID_START_TOKEN,  # noqa: E402
                         DEFAULT_VIDEO_PATCH_TOKEN)
from .multimodal_projector.builder import build_vision_projector  # noqa: E402


class VisionConfig:
    def __init__(self, frame_size=224, patch_size=14, hidden_size=1024):
        self.frame_size = frame_size
        self.patch_size = patch_size
        self.hidden_size = hidden_size
        self.use_vid_start_end = None
        self.vid_start_token = None
        self.vid_end_token = None
        self.vid_patch_token = None


_CLIP_DEFAULTS = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                      image_size=224, patch_size=14, layer_norm_eps=1e-5, hidden_act="quick_gelu")


def _clip_config(src) -> SimpleNamespace:
    """CLIP vision config from a dict, an object with attributes, or a directory with config.json."""
    d = dict(_CLIP_DEFAULTS)
    if src is None:
        pass
    elif isinstance(src, dict):
        d.update(src.get("vision_config", src))
    elif isinstance(src, str):
        path = os.path.join(src, "config.json")
        if not os.path.exists(path):
            raise FileNotFoundError(f"mm_vision_tower='{src}' must be a local directory with config.json "
                                    "(no network access on this path)")
        j = json.load(open(path))
        d.update(j.get("vision_config", j))
    else:
        for k in d:
            if hasattr(src, k):
                d[k] = getattr(src, k)
    if d["hidden_act"] != "quick_gelu":
        raise ValueError("libvcl implements the quick_gelu ViT MLP only")
    return SimpleNamespace(**d)


class VideoChatGPTConfig:
    """LLaMA config + the multimodal fields the reference adds (model_type 'VideoChatGPT')."""
    model_type = "VideoChatGPT"

    def __init__(self, **kw):
        self.hidden_size = kw.pop("hidden_size", 4096)
        self.intermediate_size = kw.pop("intermediate_size", 11008)
        self.num_hidden_layers = kw.pop("num_hidden_layers", 32)
        self.num_attention_heads = kw.pop("num_attention_heads", 32)
        self.num_key_value_heads = kw.pop("num_key_value_heads", self.num_attention_heads)
        self.vocab_size = kw.pop("vocab_size", 32000)
        self.rms_norm_eps = kw.pop("rms_norm_eps", 1e-5)
        self.rope_theta = kw.pop("rope_theta", 10000.0)
        self.max_position_embeddings = kw.pop("max_position_embeddings", 2048)
        self.use_cache = kw.pop("use_cache", True)
        for k, v in kw.items():          # mm_vision_tower, use_mm_proj, mm_hidden_size, mm_projector_type, ...
            setattr(self, k, v)
        if self.num_key_value_heads != self.num_attention_heads:
            raise ValueError("libvcl implements multi-head attention only (kv heads == heads), as Vicuna uses")

    @classmethod
    def from_pretrained(cls, path, **kw):
        j = json.load(open(os.path.join(path, "config.json")))
        j.update(kw)
        return cls(**j)


def _mask_bool(attention_mask, shape) -> torch.Tensor:
    """HF attention_mask ([B, S], bool or integer 0/1) -> a bool tensor on the host; ValueError otherwise"""
    m = torch.as_tensor(attention_mask).detach().cpu()
    B, S = int(shape[0]), int(shape[1])
    if tuple(m.shape) != (B, S):
        raise ValueError(f"attention_mask has shape {tuple(m.shape)}, input_ids {(B, S)}")
    if m.dtype != torch.bool:
        if m.is_floating_point() or m.is_complex() or not bool(((m == 0) | (m == 1)).all()):
            raise ValueError("attention_mask must be bool or integer 0/1")
        m = m != 0
    return m


def score_padding(attention_mask, labels, shape, vocab: int) -> list | None:
    """Host-side checks of forward(labels=...), before any device work. labels [B, S] must hold ids in
    [0, vocab) or -100 (IGNORE_INDEX). The mask may be left padding (-> the B pad counts, the padded prefill) or
    right padding, the layout of train.py's collator (pad_sequence with labels padded by -100) -> None: the batch
    runs unpadded, which under causal attention gives every real column exactly what its row alone gives.
    Every pad column must be labelled -100; with left padding so must the first real token, since no real position
    predicts it. Raises ValueError otherwise."""
    B, S = int(shape[0]), int(shape[1])
    lab = torch.as_tensor(labels).detach().cpu()
    if tuple(lab.shape) != (B, S):
        raise ValueError(f"labels have shape {tuple(lab.shape)}, input_ids {(B, S)}")
    if lab.is_floating_point() or lab.is_complex() or lab.dtype == torch.bool:
        raise ValueError(f"labels must be integer ids, got {lab.dtype}")
    lab = lab.to(torch.int64)
    bad = ~(((lab >= 0) & (lab < vocab)) | (lab == -100))
    if bool(bad.any()):
        b, s = (int(i) for i in bad.nonzero()[0])
        raise ValueError(f"labels[{b}, {s}] = {int(lab[b, s])} is neither a token id in [0, {vocab}) nor -100")
    if attention_mask is None:
        return None
    m = _mask_bool(attention_mask, shape)
    pads, right = [], False
    for b in range(B):
        row = m[b]
        n_real = int(row.sum())
        if n_real == 0:
            raise ValueError(f"attention_mask row {b} has no real token")
        if bool(row[S - n_real:].all()):
            pads.append(S - n_real)                     # left padding (or none)
        elif bool(row[:n_real].all()):
            pads.append(0)                              # right padding
            right = True
        else:
            raise ValueError(f"attention_mask row {b} has holes: only left or right padding is supported")
    if right and any(pads):
        raise ValueError("attention_mask mixes left- and right-padded rows")
    need_ignore = ~m
    for b, n in enumerate(pads):
        if n > 0:
            need_ignore[b, n] = True
    if bool((lab[need_ignore] != -100).any()):
        b, s = (int(i) for i in (need_ignore & (lab != -100)).nonzero()[0])
        raise ValueError(f"labels[{b}, {s}] = {int(lab[b, s])} lies on a pad column (or, with left padding, on the "
                         "first real token, which no real position predicts): it must be -100")
    return pads if any(pads) else None


def left_padding(attention_mask, shape) -> list | None:
    """Pad count per row of a left-padded batch from its HF attention_mask ([B, S], bool or integer 0/1):
    each row must be zeros followed by ones, with at least one 1. Returns None when nothing is padded
    (an all-ones mask: the unpadded path), else the list of B pad counts. Raises ValueError otherwise;
    it runs on the host, before any device work."""
    if attention_mask is None:
        return None
    m = _mask_bool(attention_mask, shape)
    B, S = int(shape[0]), int(shape[1])
    pads = []
    for b in range(B):
        row = m[b]
        n_pad = S - int(row.sum())
        if n_pad == S:
            raise ValueError(f"attention_mask row {b} has no real token")
        if not bool(row[n_pad:].all()):
            raise ValueError(f"attention_mask row {b} is not left padding (zeros, then ones): right padding and "
                             "holes are not supported; tokenize with padding_side='left'")
        pads.append(n_pad)
    return pads if any(pads) else None


class _LazyStates:
    """Tuple-like view of hidden states; entry i is produced on first access."""

    def __init__(self, n, fn):
        self._n, self._fn, self._cache = n, fn, {}

    def __len__(self):
        return self._n

    def __getitem__(self, i):
        if isinstance(i, slice):
            return tuple(self[j] for j in range(*i.indices(self._n)))
        if i < 0:
            i += self._n
        if not 0 <= i < self._n:
            raise IndexError(i)
        if i not in self._cache:
            self._cache[i] = self._fn(i)
        return self._cache[i]


class _Engines:
    """One vcl handle per process/GPU, created when both configs are known."""

    def __init__(self):
        self.engine = None


class CLIPVisionTower:
    """The vision tower with HF's calling convention (the reference holds a bare CLIPVisionModel):

        outs = tower(pixel_values, output_hidden_states=True)
        feats = outs.hidden_states[-2][:, 1:]          # video_chatgpt/inference.py:93-94

    pixel_values: [N,3,H,W] float (normalised by the image processor) or [N,H,W,3] uint8 raw frames
    (normalised on the device). hidden_states has num_hidden_layers+1 entries like HF; entries are
    computed on access; index -1 needs the last encoder layer, which is only loaded when the tower
    was built with run_layers = num_hidden_layers (the path itself never reads it)."""

    def __init__(self, owner: "VideoChatGPTLlamaForCausalLM"):
        self._owner = owner
        self.config = owner.clip_config
        self.dtype = torch.bfloat16
        self.device = torch.device("cuda")

    def eval(self): return self
    def cuda(self, *a, **k): return self
    def half(self): return self
    def to(self, *a, **k): return self

    def load_state_dict(self, sd, strict=True):
        self._owner._clip_state = {k: v for k, v in sd.items()}
        return SimpleNamespace(missing_keys=[], unexpected_keys=[])

    @torch.no_grad()
    def __call__(self, pixel_values, output_hidden_states=True, **kw):
        eng = self._owner._ensure_engine(need_clip=True)
        n_states = self.config.num_hidden_layers + 1
        px = pixel_values.cuda()

        def state(i):
            if i > eng.cfg.clip_layers:
                raise vn.VclError(f"hidden_states[{i}] needs encoder layer {i}; only {eng.cfg.clip_layers} layers are "
                                  "loaded (the path consumes hidden_states[-2])")
            return eng.clip_encode(px, n_layers=i)

        hs = _LazyStates(n_states, state)
        return SimpleNamespace(hidden_states=hs if output_hidden_states else None)

    forward = __call__


class VideoChatGPTLlamaModel:
    def __init__(self, owner, config):
        self._owner = owner
        self.config = config
        if hasattr(config, "mm_vision_tower") or owner.clip_config is not None:
            cc = owner.clip_config
            self.vision_config = VisionConfig(cc.image_size, cc.patch_size, cc.hidden_size)
        if getattr(config, "use_mm_proj", False):
            if not hasattr(config, "mm_hidden_size"):
                config.mm_hidden_size = self.vision_config.hidden_size
            if self.vision_config.frame_size == 224:       # LLaVA-v1.1-Lightning: plain linear
                config.mm_projector_type = "linear"
            self.mm_projector = build_vision_projector(config)

    def initialize_vision_modules(self, pretrain_mm_mlp_adapter=None, tune_mm_mlp_adapter=False):
        vc = self.vision_config
        self.config.use_mm_proj = True
        self.config.mm_hidden_size = vc.hidden_size
        if not hasattr(self, "mm_projector"):
            if vc.frame_size == 224:
                self.config.mm_projector_type = "linear"
            self.mm_projector = build_vision_projector(self.config)
        if pretrain_mm_mlp_adapter is not None:
            w = torch.load(pretrain_mm_mlp_adapter, map_location="cpu")
            self._owner.load_state_dict({k: v for k, v in w.items() if "mm_projector" in k}, strict=False)
        return dict(num_patches=(vc.frame_size // vc.patch_size) ** 2, vision_config=vc)


class VideoChatGPTLlamaForCausalLM:
    config_class = VideoChatGPTConfig

    def __init__(self, config: VideoChatGPTConfig, clip_config=None, max_batch: int = 1, max_seq: int | None = None,
                 clip_run_layers: int | None = None, llm_weight_format: str = "bf16", max_slots: int | None = None,
                 kv_blocks: int | None = None):
        """llm_weight_format: "bf16", or "fp8_e4m3" to hold the language model's streamed matrices as E4M3 codes
        with power-of-two row scales (vcl_load_llm_weights_ex): decode reads half the weight bytes, and every
        output is that of the bf16 engine on the dequantized weights.
        max_slots: the KV-cache slots generate_requests keeps in flight, 1 .. min(max_batch, 64); None means
        min(max_batch, 16). A capacity only: which decode kernel runs depends on the clip count of each call.
        kv_blocks: None keeps the contiguous KV cache (every slot holds max_seq columns). An int >= 2 makes the cache
        PAGED: a pool of kv_blocks blocks of 128 columns (vcl_config.kv_blocks), which the running requests of
        generate_requests take as they grow; block 0 is the park block, so kv_blocks - 1 are usable. A paged model
        serves generate_requests only (generate / forward / generate_continue raise NotImplementedError), with
        prompts of at most 512 tokens, and returns exactly what the contiguous model returns."""
        vn.weight_format_code(llm_weight_format)          # ValueError before anything else
        self._kv_blocks = vn.check_kv_blocks(kv_blocks)
        self.last_kv_stats = None
        self.last_logprobs = None      # generate / generate_continue / generate_requests(logprobs=...): per row or request
        self._pads = None              # the left padding of the last generate (log-prob positions of generate_continue)
        self._sessions: dict = {}      # kept conversations of generate_requests (paged): key -> _schedule_paged's state
        self._session_clock = 0        # last-use stamps of the kept conversations (the least recent is swapped first)
        self._n_slots = vn.slot_capacity(max_batch, max_slots)
        self._max_slots = 0 if max_slots is None else self._n_slots
        self._llm_weight_format = llm_weight_format
        self.config = config
        self.clip_config = _clip_config(clip_config if clip_config is not None
                                        else getattr(config, "mm_vision_tower", None))
        self.model = VideoChatGPTLlamaModel(self, config)
        self._state: dict = {}
        self._clip_state: dict | None = None
        self._engine = None
        self._max_batch = max_batch
        self._max_seq = max_seq or config.max_position_embeddings
        self._clip_run_layers = clip_run_layers
        self._pos = 0              # tokens in the KV cache after the last forward
        self.training = False
        self.dtype = torch.bfloat16
        self.device = torch.device("cuda")

    # ---- construction / state -----------------------------------------------------------
    @classmethod
    def from_pretrained(cls, model_name, **kw):
        """Local directory with config.json and *.safetensors / pytorch_model*.bin (no hub access)."""
        kw.pop("low_cpu_mem_usage", None); kw.pop("torch_dtype", None)
        use_cache = kw.pop("use_cache", True)
        config = VideoChatGPTConfig.from_pretrained(model_name, use_cache=use_cache)
        m = cls(config, **kw)
        files = sorted(f for f in os.listdir(model_name) if f.endswith((".safetensors", ".bin")) and "training" not in f)
        if not files:
            raise FileNotFoundError(f"no weight files in {model_name}")
        for f in files:
            path = os.path.join(model_name, f)
            if f.endswith(".safetensors"):
                from safetensors.torch import load_file
                m.load_state_dict(load_file(path), strict=False)
            else:
                m.load_state_dict(torch.load(path, map_location="cpu"), strict=False)
        return m

    def get_model(self): return self.model
    def get_vision_tower(self): return CLIPVisionTower(self)
    def eval(self): return self
    def cuda(self, *a, **k): return self
    def half(self): return self
    def to(self, *a, **k): return self
    def parameters(self): return iter(self._state.values())

    def state_dict(self):
        return dict(self._state)

    def load_state_dict(self, sd, strict=True):
        if self._engine is not None:
            raise vn.VclError("weights are already resident in libvcl; load_state_dict must precede the first forward")
        known = lambda k: k.startswith(("model.", "lm_head."))
        unexpected = [k for k in sd if not known(k)]
        for k, v in sd.items():
            if known(k):
                self._state[k] = v
        if strict and unexpected:
            raise RuntimeError(f"Unexpected key(s) in state_dict: {unexpected}")
        return SimpleNamespace(missing_keys=[], unexpected_keys=unexpected)

    def resize_token_embeddings(self, n: int):
        """Grow embed_tokens / lm_head to n rows; new rows start as the mean of the old ones (HF's
        mean-resizing default) and are normally overwritten by the projection checkpoint that the
        reference loads right after (eval/model_utils.py:119-127)."""
        for key in ("model.embed_tokens.weight", "lm_head.weight"):
            w = self._state.get(key)
            if w is None or w.shape[0] == n:
                continue
            if w.shape[0] > n:
                self._state[key] = w[:n].clone()
            else:
                extra = w.float().mean(0, keepdim=True).to(w.dtype).expand(n - w.shape[0], -1)
                self._state[key] = torch.cat([w, extra], 0)
        self.config.vocab_size = n

    def initialize_vision_tokenizer(self, mm_use_vid_start_end, tokenizer, device=None,
                                    tune_mm_mlp_adapter=False, pretrain_mm_mlp_adapter=None):
        vc = self.get_model().vision_config
        vc.use_vid_start_end = mm_use_vid_start_end
        tokenizer.add_tokens([DEFAULT_VIDEO_PATCH_TOKEN], special_tokens=True)
        self.resize_token_embeddings(len(tokenizer))
        if mm_use_vid_start_end:
            tokenizer.add_tokens([DEFAULT_VID_START_TOKEN, DEFAULT_VID_END_TOKEN], special_tokens=True)
            self.resize_token_embeddings(len(tokenizer))
            vc.vid_start_token, vc.vid_end_token = tokenizer.convert_tokens_to_ids(
                [DEFAULT_VID_START_TOKEN, DEFAULT_VID_END_TOKEN])
        vc.vid_patch_token = tokenizer.convert_tokens_to_ids([DEFAULT_VIDEO_PATCH_TOKEN])[0]

    # ---- engine ---------------------------------------------------------------------------
    def _ensure_engine(self, need_clip=False, need_llm=False):
        if self._engine is None:
            c, cc = self.config, self.clip_config
            k = vn.vcl_config()
            k.clip_layers = cc.num_hidden_layers - 1 if self._clip_run_layers is None else self._clip_run_layers
            k.clip_hidden, k.clip_inter, k.clip_heads = cc.hidden_size, cc.intermediate_size, cc.num_attention_heads
            k.image_size, k.patch_size, k.clip_ln_eps = cc.image_size, cc.patch_size, cc.layer_norm_eps
            k.llm_layers, k.llm_hidden, k.llm_inter = c.num_hidden_layers, c.hidden_size, c.intermediate_size
            k.llm_heads, k.vocab = c.num_attention_heads, c.vocab_size
            k.rms_eps, k.rope_theta = c.rms_norm_eps, c.rope_theta
            kind = getattr(c, "mm_projector_type", "linear")
            k.proj_type = vn.PROJ_LINEAR if kind == "linear" else vn.PROJ_MLP2X_GELU
            k.n_temporal = 100
            k.max_frames, k.max_batch, k.max_seq = 100, self._max_batch, self._max_seq
            k.max_slots = self._max_slots
            # a paged cache is the trailing vcl_config.kv_blocks (vcl_native.vcl_config_ex)
            self._engine = vn.Engine(k, kv_blocks=self._kv_blocks) if self._kv_blocks else vn.Engine(k)
            self._clip_loaded = self._llm_loaded = False
        if need_clip and not self._clip_loaded:
            if not self._clip_state:
                raise vn.VclError("vision tower weights were never loaded (CLIPVisionTower.load_state_dict)")
            self._engine.load_clip(self._clip_state)
            self._clip_state, self._clip_loaded = None, True
        if need_llm and not self._llm_loaded:
            self._engine.load_llm(self._state, weight_format=self._llm_weight_format)
            self._llm_loaded = True
        return self._engine

    # ---- validation (same errors as video_chatgpt.py:119-128,150-157) ---------------------
    def _video_spans(self, input_ids: torch.Tensor, n_vid: int, n_pad: list | None = None) -> list:
        """Index of the row after which the projected video rows are spliced, per sample (-1: none).
        n_pad: left padding per row; a video span must lie inside the real tokens."""
        vc = self.get_model().vision_config
        ids = input_ids.cpu()
        starts = []
        for b, row in enumerate(ids):
            if (row == vc.vid_patch_token).sum() == 0:
                starts.append(vn.NO_VIDEO)             # text-only sample
                continue
            if vc.use_vid_start_end:
                if (row == vc.vid_start_token).sum() != (row == vc.vid_end_token).sum():
                    raise ValueError("The number of video start tokens and video end tokens should be the same.")
                pos = torch.where(row == vc.vid_start_token)[0]
                if len(pos) != 1:
                    raise ValueError("libvcl supports exactly one video span per sample")
                s = int(pos[0])
                if s + n_vid + 1 >= len(row) or row[s + n_vid + 1] != vc.vid_end_token:
                    raise ValueError("The video end token should follow the video start token.")
                starts.append(s)
            else:
                if (row == vc.vid_patch_token).sum() != n_vid:
                    raise ValueError("The number of video patch tokens should be the same as the number of video patches.")
                idx = torch.where(row == vc.vid_patch_token)[0]
                s0 = int(idx[0])
                if (idx != torch.arange(s0, s0 + n_vid)).any():
                    raise ValueError("The video patch tokens should be consecutive.")
                starts.append(s0 - 1)                  # rows s0 .. s0+n_vid-1 are replaced (-1: from row 0)
            first = starts[-1] + (0 if vc.use_vid_start_end else 1)      # first column of the span
            if n_pad is not None and first < n_pad[b]:
                raise ValueError(f"sample {b}: the video span starts at column {first}, inside the left padding "
                                 f"({n_pad[b]} columns)")
        return starts

    def _spans_dev(self, ids, feats, n_vid, n_pad=None):
        starts = self._video_spans(ids, n_vid, n_pad) if feats is not None else [vn.NO_VIDEO] * ids.shape[0]
        return torch.tensor(starts, dtype=torch.int32, device="cuda")

    # ---- forward / generate ----------------------------------------------------------------
    def _not_paged(self, what):
        if self._kv_blocks:
            raise NotImplementedError(f"{what}: this model has a paged KV cache (kv_blocks={self._kv_blocks}), which "
                                      "serves generate_requests only")

    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, past_key_values=None, inputs_embeds=None, labels=None,
                use_cache=None, output_attentions=None, output_hidden_states=None,
                video_spatio_temporal_features=None, return_dict=None, logits_to_keep=1):
        """logits_to_keep (transformers 5.x's name): 1, the default, returns the last position's logits [B,1,V];
        0 returns every position's [B,S,V]. labels [B,S] (train.py's IGNORE_INDEX -100 on prompt and padding)
        returns the reference's loss, a 0-d bf16 tensor, with the logits of every position (vcl_llm_score)."""
        self._not_paged("forward")
        if inputs_embeds is not None or output_attentions:
            raise NotImplementedError("inference path only: input_ids in, logits out")
        if logits_to_keep not in (0, 1):
            raise NotImplementedError(f"logits_to_keep={logits_to_keep}: only 1 (last position) and 0 (all positions)")
        B, S = input_ids.shape
        cached_step = S == 1 and past_key_values is not None
        if labels is not None or (logits_to_keep == 0 and not cached_step):
            return self._score(input_ids, attention_mask, labels, cached_step, output_hidden_states,
                               video_spatio_temporal_features)
        # a cached step ignores the mask: the KV cache carries the padding of its prefill
        pads = None if cached_step else left_padding(attention_mask, (B, S))
        if pads is not None and output_hidden_states:
            raise NotImplementedError("output_hidden_states is not supported with a padded attention_mask")
        eng = self._ensure_engine(need_llm=True)
        ids = input_ids.cuda().to(torch.int64)
        if cached_step:
            # cached single-token step: the video features are ignored, as in the reference (:103)
            logits, _ = eng.decode_step(ids[:, 0].to(torch.int32).contiguous(), self._pos, want_logits=True)
            self._pos += 1
            hs = None
        else:
            feats = video_spatio_temporal_features
            vs = self._spans_dev(ids, feats, eng.NV, pads)
            if feats is not None:
                feats = feats.cuda()
            hs = None
            if output_hidden_states:
                # HF's tuple: [0] the spliced input embeddings, [i] the output of layer i, and the
                # LAST entry after the final RMSNorm ($TF/models/llama/modeling_llama.py:411-425)
                states, logits = eng.prefill_states(ids, feats, vs, want_logits=True)
                L, D = self.config.num_hidden_layers, self.config.hidden_size
                norm_w = self._state["model.norm.weight"].to(device="cuda", dtype=torch.bfloat16).contiguous()
                last = vn.op_rmsnorm(states[L].reshape(B * S, D), norm_w, self.config.rms_norm_eps).view(B, S, D)
                hs = tuple(states[i] for i in range(L)) + (last,)
            else:
                _, logits, _ = eng.prefill(ids, feats, vs, want_logits=True, want_token=False, n_pad=pads)
            self._pos = S
        return SimpleNamespace(loss=None, logits=logits.to(torch.bfloat16)[:, None, :], past_key_values=self._pos,
                               hidden_states=hs, attentions=None)

    __call__ = forward

    def _score(self, input_ids, attention_mask, labels, cached_step, output_hidden_states, feats):
        """forward with labels and / or every position's logits: one vcl_llm_score call"""
        if cached_step:
            raise NotImplementedError("labels on a cached single-token step are not supported")
        if output_hidden_states:
            raise NotImplementedError("output_hidden_states together with labels or logits_to_keep=0 is not supported")
        B, S = input_ids.shape
        if labels is not None:
            pads = score_padding(attention_mask, labels, (B, S), self.config.vocab_size)
        else:
            pads = left_padding(attention_mask, (B, S))
        eng = self._ensure_engine(need_llm=True)
        ids = input_ids.cuda().to(torch.int64)
        vs = self._spans_dev(ids, feats, eng.NV, pads)
        if feats is not None:
            feats = feats.cuda()
        lab = None if labels is None else torch.as_tensor(labels).cuda().to(torch.int64)
        logits, _, loss = eng.score(ids, feats, vs, labels=lab, n_pad=pads, want_logits=True)
        self._pos = S
        return SimpleNamespace(loss=None if loss is None else loss.to(torch.bfloat16), logits=logits,
                               past_key_values=self._pos, hidden_states=None, attentions=None)

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, attention_mask=None,
                                      inputs_embeds=None, **kwargs):
        """Same contract as the reference (:253-273), with the cache test made explicit: only a
        NON-EMPTY cache narrows input_ids to the last token (the reference's truthiness test breaks
        under transformers 5.x, SURVEY.md 8c)."""
        if past_key_values:
            input_ids = input_ids[:, -1:]
        return {"input_ids": input_ids, "past_key_values": past_key_values, "use_cache": kwargs.get("use_cache"),
                "attention_mask": attention_mask,
                "video_spatio_temporal_features": kwargs.get("video_spatio_temporal_features")}

    _GREEDY_CHUNK = 32      # tokens per device-side decode loop between two host-side EOS checks

    def _eos_pad(self, eos_token_id, pad_token_id):
        """HF generate's defaults: eos from the (generation) config -- LLaMA / Vicuna: 2 -- and padding
        of finished rows with pad_token_id, which falls back to the eos id. Pass eos_token_id=None to
        decode a fixed number of tokens (the benchmark does)."""
        if eos_token_id == "config":
            eos_token_id = getattr(self.config, "eos_token_id", 2)
            if isinstance(eos_token_id, (list, tuple)):
                eos_token_id = eos_token_id[0] if eos_token_id else None
        if pad_token_id is None:
            pad_token_id = getattr(self.config, "pad_token_id", None)
        if pad_token_id is None:
            pad_token_id = eos_token_id
        return eos_token_id, pad_token_id

    @staticmethod
    def _sampling_args(temperature, top_k, seed, what="generate"):
        """Checks the settings of the device sampler on the host -> (temperature, top_k, seed mod 2**64)"""
        t = float(temperature)
        if not math.isfinite(t) or t < 0:
            raise ValueError(f"{what}: temperature {temperature} must be a finite value >= 0")
        k = 0 if top_k is None else top_k
        if isinstance(k, bool) or not isinstance(k, int) or k < 0:
            raise ValueError(f"{what}: top_k {top_k} must be an int >= 0 (0 or None: every token)")
        if seed is not None and (isinstance(seed, bool) or not isinstance(seed, int)):
            raise ValueError(f"{what}: seed {seed!r} must be an int")
        return t, k, None if seed is None else seed % 2 ** 64

    def _nucleus_args(self, top_p, repetition_penalty, what="generate", sampled=True, device=True):
        """Checks top_p and repetition_penalty on the host -> (top_p, repetition_penalty) as floats; 1.0 is off. The
        device sampler's vocabulary limit applies when the call runs there (`device`) and turns a setting on: the
        penalty, or top_p on a `sampled` call (a greedy one ignores top_p, as HF does)."""
        p, r = float(top_p), float(repetition_penalty)
        if not 0.0 <= p <= 1.0:
            raise ValueError(f"{what}: top_p {top_p} must lie in [0, 1] (1: off)")
        if not math.isfinite(r) or r <= 0:
            raise ValueError(f"{what}: repetition_penalty {repetition_penalty} must be a finite value > 0 (1: off)")
        V = self.config.vocab_size
        if device and (r != 1.0 or (sampled and p != 1.0)) and V > vn.SAMPLE_WIDE_MAX_V:
            raise ValueError(f"{what}: top_p and repetition_penalty take a vocabulary of at most {vn.SAMPLE_WIDE_MAX_V} "
                             f"tokens on the device sampler, this model has {V}")
        return p, r

    @staticmethod
    def _set_entries(eng, clips, temperature, top_k, seeds, top_p, penalty):
        """One sampling-table write: set_sampling when every entry has top_p 1 and penalty 1 (what a call without
        them always made), set_sampling_ex otherwise"""
        if all(p == 1.0 for p in top_p) and all(r == 1.0 for r in penalty):
            eng.set_sampling(clips, temperature, top_k, seeds)
        else:
            eng.set_sampling_ex(clips, temperature, top_k, seeds, top_p, penalty)

    @contextlib.contextmanager
    def _sampling(self, eng, clips, temperature, top_k, seeds, top_p=1.0, penalty=1.0):
        """Entries `clips` of the engine's sampling table sample (temperature 0: greedy, with the penalty) for the
        duration of the block and are greedy, without top-p or penalty, again afterwards, also when the block raises."""
        n = len(clips)
        self._set_entries(eng, clips, temperature, top_k, seeds, [top_p] * n, [penalty] * n)
        try:
            yield
        finally:
            eng.set_sampling(clips, [0.0] * n, [0] * n, [0] * n)

    @staticmethod
    def _token_sets(eng, rows):
        """(entry, ids) pairs: each entry's token set of the repetition penalty becomes its ids, one call each"""
        for b, ids in rows:
            eng.set_token_set(b, ids)

    @staticmethod
    def _logprobs_arg(v, what):
        """Checks a logprobs setting on the host: None (off) or an int 0 .. vn.LOGPROBS_MAX"""
        if v is None:
            return None
        if isinstance(v, bool) or not isinstance(v, int) or not 0 <= v <= vn.LOGPROBS_MAX:
            raise ValueError(f"{what}: logprobs {v!r} must be None or an int 0..{vn.LOGPROBS_MAX} (the alternatives "
                             "reported per token besides the chosen one)")
        return v

    @contextlib.contextmanager
    def _logprobs(self, eng, clips, top_n):
        """Entries `clips` report top_n alternatives (None: nothing changes) for the duration of the block and are off
        again afterwards, also when the block raises."""
        if top_n is None:
            yield
            return
        eng.set_logprobs(clips, [top_n] * len(clips))
        try:
            yield
        finally:
            eng.set_logprobs(clips, [-1] * len(clips))

    @staticmethod
    def _logprob_entry(ids, lp, k):
        """host rows ids / lp [n, 1 + LOGPROBS_MAX] -> one entry of last_logprobs"""
        return dict(token_logprobs=lp[:, 0].clone(), top_ids=ids[:, 1:1 + k].to(torch.int64),
                    top_logprobs=lp[:, 1:1 + k].clone())

    def _read_logprobs(self, eng, new, p0, k, eos):
        """last_logprobs of a static batch: row b's new tokens new[b] [n] took positions p0[b] .. p0[b] + n - 1 of
        entry b. Positions after a row's first EOS (its padding) hold NaN / -1."""
        B, n = new.shape
        out = []
        for b in range(B):
            ids, lp = eng.read_logprobs(b, p0[b], n)
            e = self._logprob_entry(ids.cpu(), lp.cpu(), k)
            hit = (new[b] == eos).nonzero() if eos is not None else []
            if len(hit):
                f = int(hit[0]) + 1
                e["token_logprobs"][f:] = float("nan")
                e["top_ids"][f:] = -1
                e["top_logprobs"][f:] = float("nan")
            out.append(e)
        return out

    @torch.no_grad()
    def generate(self, input_ids, video_spatio_temporal_features=None, do_sample=False, temperature=1.0,
                 max_new_tokens=32, stopping_criteria=None, eos_token_id="config", pad_token_id=None, top_k=50,
                 attention_mask=None, seed=None, logprobs=None, top_p=1.0, repetition_penalty=1.0, **kw):
        """Returns [B, S+n] int64 INCLUDING the prompt, like HF generate (inference.py:105-120), and
        like HF it stops at EOS (config.eos_token_id unless eos_token_id is given; None disables it):
        finished rows are padded, the call returns when every row has finished.
        Greedy decoding without stopping criteria runs on the device: prefill + CUDA-graph decode
        loops of 32 tokens with one host-side EOS check per loop (a single loop of exactly
        max_new_tokens when EOS is disabled). Sampling (temperature, top-k 50 as HF defaults) or
        stopping criteria take one C-ABI step per token with the host-side check the reference also
        performs every step.
        attention_mask [B, S]: a left-padded batch of prompts of different lengths (module docstring); every
        path continues the padding through its decode steps. An all-ones mask is the same as none.
        seed (an int): do_sample=True samples ON THE DEVICE (vcl_llm_set_sampling) with the same temperature /
        top-k rules, row b with seed + b (mod 2**64), through the prefill and the CUDA-graph loops; EOS, padding
        and stopping criteria are applied on the host between loops of _GREEDY_CHUNK tokens, token by token as
        the stepwise path does. Each row's tokens depend on its seed and positions only. Without a seed,
        do_sample=True keeps the stepwise path and torch's RNG (torch.manual_seed).
        logprobs (an int 0 .. 20): self.last_logprobs gets, per row, the log-probabilities of its new tokens as
        compute_transition_scores(normalize_logits=True) gives them on HF's scores (DESIGN.md section 3):
        token_logprobs f32 [n_new], and the `logprobs` most likely tokens of each step, top_ids int64 [n_new, k] and
        top_logprobs f32 [n_new, k]; positions after a row's EOS hold NaN / -1. They are computed on the device next
        to the token, so greedy calls take the device loops (the seeded path's, with greedy entries) and return the
        same tokens; unseeded sampling cannot report them (NotImplementedError: pass seed=).
        top_p (1.0: off) and repetition_penalty (1.0: off): HF's TopPLogitsWarper and RepetitionPenaltyLogitsProcessor,
        in HF's order (penalty, temperature, top-k, top-p; DESIGN.md section 3). The penalty divides (multiplies, when
        negative) the logits of every token of the row's input_ids so far (prompt, padding, new tokens); top-p only
        applies when sampling. Seeded sampling applies both on the device; a greedy call with a penalty takes the
        device loops with greedy entries; unseeded sampling applies them on the host, step by step, as HF does."""
        self._not_paged("generate")
        lp_n = self._logprobs_arg(logprobs, "generate")
        if lp_n is not None and do_sample and seed is None:
            raise NotImplementedError("generate: logprobs are computed by the device sampler, and sampling there needs "
                                      "seed= (unseeded do_sample=True draws from torch's RNG on the host)")
        top_p, penalty = self._nucleus_args(top_p, repetition_penalty, "generate", do_sample,
                                            device=not do_sample or seed is not None)
        seeded = do_sample and seed is not None
        if seeded:
            temperature, top_k, seed = self._sampling_args(temperature, top_k, seed)
        pads = left_padding(attention_mask, input_ids.shape)
        self.last_logprobs = None
        eng = self._ensure_engine(need_llm=True)
        ids = input_ids.cuda().to(torch.int64)
        B, S = ids.shape
        feats = video_spatio_temporal_features
        vs = self._spans_dev(ids, feats, eng.NV, pads)
        if feats is not None:
            feats = feats.cuda()
        n = min(max_new_tokens, self._max_seq - S)
        if n <= 0:
            raise ValueError(f"prompt length {S} leaves no room in max_seq {self._max_seq}")
        eos, pad = self._eos_pad(eos_token_id, pad_token_id)
        self._pads = pads
        if seeded or lp_n is not None or (penalty != 1.0 and not do_sample):
            clips = list(range(B))
            if seeded:
                samp = self._sampling(eng, clips, [temperature] * B, [top_k] * B, [seed + b for b in clips], top_p,
                                      penalty)
            elif penalty != 1.0:   # greedy entries with the penalty
                samp = self._sampling(eng, clips, [0.0] * B, [0] * B, [0] * B, 1.0, penalty)
            else:
                samp = contextlib.nullcontext()
            if penalty != 1.0:
                self._token_sets(eng, [(b, ids[b]) for b in clips])
            with samp, self._logprobs(eng, clips, lp_n):
                if eos is None and not stopping_criteria:
                    new = eng.generate(ids, feats, vs, n, n_pad=pads)
                    self._pos = S + n - 1
                    self._last_out = torch.cat([ids, new.to(torch.int64)], dim=1)
                else:
                    first = eng.generate(ids, feats, vs, min(n, self._GREEDY_CHUNK), n_pad=pads)
                    self._last_out = self._host_stops(eng, ids, first, n, stopping_criteria, eos, pad)
            if lp_n is not None:   # the token after the prompt takes position S - n_pad[b]
                self.last_logprobs = self._read_logprobs(eng, self._last_out[:, S:].cpu(),
                                                         [S - (pads[b] if pads else 0) for b in range(B)], lp_n, eos)
            return self._last_out
        if do_sample or stopping_criteria:
            _, logits, _ = eng.prefill(ids, feats, vs, want_logits=True, want_token=False, n_pad=pads)
            self._pos = S
            self._last_out = self._stepwise(eng, ids, logits, n, do_sample, temperature, stopping_criteria, eos, pad,
                                            top_k, top_p, penalty)
            return self._last_out
        if eos is None:
            new = eng.generate(ids, feats, vs, n, n_pad=pads).to(torch.int64)
            self._pos = S + n - 1
            self._last_out = torch.cat([ids, new], dim=1)
            return self._last_out
        # greedy with EOS: device loops of _GREEDY_CHUNK tokens, EOS looked for between them
        c = min(n, self._GREEDY_CHUNK)
        new = eng.generate(ids, feats, vs, c, n_pad=pads).to(torch.int64)
        while True:
            new, done = self._mask_finished(new, eos, pad)
            k = new.shape[1]
            if done or k >= n:
                break
            m = min(self._GREEDY_CHUNK, n - k)
            more = eng.decode_loop(new[:, -1].to(torch.int32).contiguous(), S + k - 1, m + 1)   # padding continues
            new = torch.cat([new, more[:, 1:].to(torch.int64)], dim=1)
        self._pos = S + new.shape[1] - 1
        self._last_out = torch.cat([ids, new], dim=1)
        return self._last_out

    def _host_stops(self, eng, out, new, n, stopping_criteria, eos, pad):
        """The device-sampled loop of generate / generate_continue: `new` [B, c] int32 holds the first c tokens
        after the context `out` [B, L] (the first at column L). _stepwise's EOS / padding / stopping-criteria
        logic runs token by token over each chunk on the host; the device decodes the next _GREEDY_CHUNK tokens
        from the last kept (padded) token until a rule stops or n tokens are out. Returns [B, L + k]; self._pos
        ends at L + k - 1, where _stepwise leaves it (columns decoded past the stop are overwritten by a
        continuation). The sequence lives in one [B, L + n] buffer on out's device, filled by one copy per chunk;
        a stopping criterion is called with a view of its first L + j columns, so a call costs no copy."""
        dev, (B, L) = out.device, out.shape
        full = torch.empty(B, L + n, dtype=torch.int64, device=dev)
        full[:, :L] = out
        unfinished = [True] * B
        k = 0                                   # tokens kept so far
        while True:
            chunk, done, eos_stop = [], False, False
            for col in zip(*new.tolist()):
                if eos is not None:
                    col = [t if u else pad for t, u in zip(col, unfinished)]
                    unfinished = [u and t != eos for t, u in zip(col, unfinished)]
                chunk.append(col)
                if eos is not None and not any(unfinished):
                    done = eos_stop = True
                    break
                if k + len(chunk) == n:
                    done = True
                    break
            full[:, L + k:L + k + len(chunk)] = torch.tensor(chunk, dtype=torch.int64).T.to(dev)
            if stopping_criteria:
                # as in _stepwise: the criteria are not asked about the step at which every row has reached EOS
                for j in range(len(chunk) - (1 if eos_stop else 0)):
                    if any(c(full[:, :L + k + j + 1], None) for c in stopping_criteria):
                        chunk, done = chunk[:j + 1], True
                        break
            k += len(chunk)
            if done:
                break
            m = min(self._GREEDY_CHUNK, n - k)
            last = full[:, L + k - 1].to(torch.int32).contiguous()
            new = eng.decode_loop(last, L + k - 1, m + 1)[:, 1:]
        self._pos = L + k - 1
        return full[:, :L + k].clone()

    @staticmethod
    def _mask_finished(new, eos, pad):
        """Pad every row after its first EOS; when all rows have one, cut at the longest row."""
        is_eos = new == eos
        seen = torch.cumsum(is_eos.to(torch.int32), dim=1)
        after = (seen - is_eos.to(torch.int32)) > 0            # strictly after the first EOS
        new = torch.where(after, torch.full_like(new, pad), new)
        if bool((seen[:, -1] > 0).all()):
            first = is_eos.to(torch.int32).argmax(dim=1)
            return new[:, : int(first.max()) + 1], True
        return new, False

    # decode steps per slot_decode call of generate_requests between two host-side checks. 8 measured best with
    # tools/bench_inflight.py (64 requests, 16..384 tokens, 7B shapes, H100 at 400 W): 7.89 / 8.13 / 8.35 s for 8 /
    # 16 / 32 at 16 slots, 19.5 / 19.9 / 20.7 s at 4 -- a retired slot idles for the rest of its chunk
    _SLOT_CHUNK = 8
    # the longest prompt a packed admission (vcl_llm_slots_prefill) takes: the key limit of its attention kernel
    _PACKED_MAX_S = 512

    @torch.no_grad()
    def generate_requests(self, requests, max_new_tokens=32, eos_token_id="config", stopping_criteria=None,
                          slots=None, do_sample=False, packed_admission=False, temperature=1.0, top_k=50, seed=None,
                          chunked_prefill=False, logprobs=None, top_p=1.0, repetition_penalty=1.0):
        """Greedy generation for many independent requests by in-flight (continuous) batching: every request
        owns a slot of the KV cache while it runs, and a finished request's slot takes the next queued one at
        once while the other slots keep decoding (a static batch decodes until its longest row finishes).

        requests: each a dict with "input_ids" [S_i] or [1, S_i], optionally "video_spatio_temporal_features"
        (the pooled [100+P, 1024] features of its video), "max_new_tokens" and "stopping_criteria" (a list, e.g.
        the reference's KeywordsStoppingCriteria built for this prompt); a bare tensor is a prompt alone. The
        keyword arguments are the defaults of requests that do not set their own; a shared stopping criterion is
        called with every request's own sequence, so it must not keep per-prompt state.
        Returns a list in request order: request i's [1, S_i + n_i] int64, prompt included, as generate returns
        it for that request alone. A request ends at its first EOS, at its max_new_tokens, or at the first token
        where one of its stopping criteria fires (called token by token with the [1, S_i + k] prefix on the host,
        as a stepwise generate would call it).
        slots: cache slots in flight, default and at most the engine's slot count (max_slots; by default
        min(max_batch, 16)). Requests are admitted one prefill
        at a time; all slots then decode _SLOT_CHUNK steps per device call. Everything is validated before any
        device work. Afterwards there is no turn for generate_continue to continue; on a paged model a conversation
        continues through the sessions below.
        packed_admission: at every admission point all free slots are filled from the queue (in queue order) by
        one packed prefill (Engine.slots_prefill) instead of one prefill each; a prompt longer than
        _PACKED_MAX_S is admitted alone. The results are the same either way.
        do_sample / temperature / top_k / seed: sampling on the device, as generate(seed=...) samples. A request dict
        may set its own "do_sample", "temperature", "top_k" and "seed"; a sampled request without its own seed
        gets seed + its index (mod 2**64). Greedy and sampled requests share the batch; each admission writes the
        admitted slots' entries of the engine's sampling table with one set_sampling call, and every slot is
        greedy again when the call returns. A request's tokens depend on its seed and positions only: not on its
        slot, its neighbours, the queue order or the admission mode. Sampling without any seed is not supported
        in flight (only the stepwise generate draws from torch's RNG).
        A paged model (kv_blocks) gives each request only the 128-column blocks it has written, so the requests in
        flight follow their actual lengths: see _schedule_paged. The results are the same bit for bit; afterwards
        self.last_kv_stats holds the preemptions, the bytes swapped out and the peak blocks in use.
        chunked_prefill: on a paged model, prompts longer than _PACKED_MAX_S tokens (up to max_seq - max_new_tokens)
        are prefilled in chunks of _PACKED_MAX_S rows (_prefill_chunked) instead of being rejected; last_kv_stats
        then also counts the chunked prompts and the chunk calls. The results are those of a contiguous model.
        A contiguous model accepts the flag and ignores it: it prefills any prompt up to max_seq in one pass.
        Sessions (paged models only; a contiguous model raises ValueError). A request with "session": key (any
        hashable) starts a conversation: when it ends, its tokens [L] and the cache blocks of columns 0 .. L - 2 are
        kept under key, across calls, until end_session(key). A request with "continues": key is the next turn of
        that conversation: its input_ids are the new text only (as generate_continue's new_input_ids), only the last
        kept token and that text are prefilled (at most _PACKED_MAX_S rows), it returns the whole conversation
        [1, L + S_new + n] (which its stopping criteria see too) and the conversation stays kept under key. Every turn
        returns what generate followed by generate_continue (B = 1, same arguments) returns on a contiguous model.
        Kept conversations are swapped to host memory, least recently used first, before a running request is
        preempted (_schedule_paged). Rejected before any device work: an unknown key to continue, a session key
        already kept, a key started and continued in one call, a key continued twice in one call, video features on
        a continuation, and a continuation that overflows max_seq or the pool. last_kv_stats then also counts the
        continuations, the prefill rows they did not recompute (reused_rows), the conversations swapped out
        (session_swaps, session_swapped_bytes) and the conversations kept, resident and swapped at the end.
        logprobs (an int 0 .. 20, or a request's own "logprobs" key): self.last_logprobs[i] holds request i's
        log-probabilities as generate(logprobs=...) reports them, for its new tokens only (a continuation: this
        turn's), or None when the request did not ask. Each admission writes the admitted slots' log-prob entries
        (a slot without a request is off), and each decode chunk's rows come back in one copy; the values do not
        depend on slot, neighbours, queue order, admission mode, paging or preemption.
        top_p / repetition_penalty (1.0: off), or a request's own "top_p" / "repetition_penalty" keys: as in generate,
        on the device. top_p applies to sampled requests; the penalty to greedy and sampled ones, over the request's own
        prompt (a continuation: the whole conversation) and its new tokens. The slot's token set is written when the
        request is admitted (before each chunk of a chunked prompt) and rebuilt from the prompt and the tokens the host
        holds when it resumes after a preemption; nothing carries over from the slot's earlier requests. Requests
        without either setting write the sampling table with set_sampling and launch what they launched before."""
        self._logprobs_arg(logprobs, "generate_requests")
        for i, r in enumerate(requests):
            r = r if isinstance(r, dict) else {}
            self._logprobs_arg(r.get("logprobs", logprobs), f"request {i}")
            if not self._kv_blocks and (r.get("session") is not None or r.get("continues") is not None):
                raise ValueError(f"request {i}: conversation sessions (\"session\" / \"continues\") need a paged KV "
                                 "cache (kv_blocks=...); on this model use generate and generate_continue")
            if r.get("do_sample", do_sample) and r.get("seed", seed) is None:
                raise NotImplementedError(f"request {i}: generate_requests decodes greedily unless given a seed; "
                                          "sampling in flight needs seed= (the call's or the request's own)")
            self._nucleus_args(r.get("top_p", top_p), r.get("repetition_penalty", repetition_penalty), f"request {i}",
                               r.get("do_sample", do_sample))
        cap = self._n_slots
        n_slots = cap if slots is None else int(slots)
        if not 1 <= n_slots <= cap:
            if self._max_slots:
                raise ValueError(f"slots={slots} outside 1..{cap} (max_slots {self._max_slots})")
            raise ValueError(f"slots={slots} outside 1..{cap} (at most 16 and at most max_batch {self._max_batch})")
        eng = self._ensure_engine(need_llm=True)
        samp = dict(do_sample=do_sample, temperature=temperature, top_k=top_k, seed=seed, logprobs=logprobs, top_p=top_p,
                    repetition_penalty=repetition_penalty)
        reqs = [self._request(i, r, max_new_tokens, stopping_criteria, eng.NV, samp) for i, r in enumerate(requests)]
        if self._kv_blocks:
            self._bind_sessions(reqs)
            self._check_paged(reqs, chunked_prefill)
        sampling = any(r.temperature > 0 or r.penalty != 1.0 for r in reqs)
        eos, _ = self._eos_pad(eos_token_id, None)
        self._last_out, self._pos, self.last_logprobs = None, 0, None
        n_slots = min(n_slots, len(reqs))
        lps = _RequestLogprobs(eng, reqs, n_slots, self.device)
        try:
            if self._kv_blocks:
                out = self._schedule_paged(eng, reqs, n_slots, packed_admission, sampling, eos, chunked_prefill, lps)
            else:
                out = self._schedule(eng, reqs, n_slots, packed_admission, sampling, eos, lps)
            if lps.on:
                self.last_logprobs = lps.result()
            return out
        finally:
            if sampling:
                eng.set_sampling(list(range(n_slots)), [0.0] * n_slots, [0] * n_slots, [0] * n_slots)
            if lps.on:
                eng.set_logprobs(list(range(n_slots)), [-1] * n_slots)

    def _schedule(self, eng, reqs, n_slots, packed_admission, sampling, eos, lps=None):
        """The admission / decode loop of generate_requests"""
        lps = lps or _RequestLogprobs(eng, reqs, n_slots, self.device)
        dev = self.device
        results = [None] * len(reqs)
        queue = collections.deque(range(len(reqs)))
        owner = [None] * n_slots            # request of each slot
        pos = [0] * n_slots                 # tokens in each slot's cache; a slot without a request is parked at 0
        unseen = [False] * n_slots          # the slot's first token (from its prefill) has not reached the host yet
        gen = {}                            # request -> its new tokens so far
        first = torch.zeros(n_slots, dtype=torch.int32, device=dev)     # the token each slot is fed next
        while True:
            admitted = []
            for s in range(n_slots):
                if owner[s] is None and queue:
                    i = queue.popleft()
                    admitted.append((s, i))
                    owner[s], pos[s], unseen[s], gen[i] = i, reqs[i].S, True, []
            if admitted and sampling:
                self._admit_sampling(eng, [(s, reqs[i]) for s, i in admitted])
            lps.sync(owner)
            if admitted and packed_admission:
                self._admit_packed(eng, [(s, reqs[i]) for s, i in admitted], first)
            elif admitted:
                for s, i in admitted:
                    r = reqs[i]
                    feats = None if r.feats is None else r.feats.to(dev)
                    vs = torch.tensor([r.vid_start], dtype=torch.int32, device=dev)
                    eng.slot_prefill(s, r.ids.to(dev), feats, vs, tok_out=first[s:s + 1])
            active = [s for s in range(n_slots) if owner[s] is not None]
            if not active:
                return results
            # shorter than a chunk only when a slot nears max_seq
            m = min([self._SLOT_CHUNK] + [self._max_seq - pos[s] for s in active])
            out = eng.slot_decode(first, pos, m + 1)
            first = out[:, m].contiguous()
            host = out.tolist()
            running = [(s, owner[s]) for s in active]
            for s in active:
                i = owner[s]
                r = reqs[i]
                pos[s] += m
                for t in (host[s] if unseen[s] else host[s][1:]):
                    gen[i].append(t)
                    if self._request_done(r, gen[i], eos):
                        results[i] = torch.cat([r.ids, torch.tensor(gen[i], dtype=torch.int64)])[None].to(dev)
                        owner[s], pos[s] = None, 0
                        break
                unseen[s] = False
            lps.collect([(s, i, len(gen[i])) for s, i in running])

    def _admit_sampling(self, eng, group, resumed=()):
        """The sampling-table entries of the (slot, request) pairs admitted at one point, in one write, and the token
        set of each penalized one: its ids; for a (slot, request, tokens) of `resumed`, its ids then those tokens."""
        rows = list(group) + [(s, r) for s, r, _ in resumed]
        self._set_entries(eng, [s for s, _ in rows], [r.temperature for _, r in rows], [r.top_k for _, r in rows],
                          [r.seed for _, r in rows], [r.top_p for _, r in rows], [r.penalty for _, r in rows])
        sets = [(s, r.ids) for s, r in group if r.penalty != 1.0]
        sets += [(s, torch.cat([r.ids, torch.tensor(toks, dtype=torch.int64)])) for s, r, toks in resumed
                 if r.penalty != 1.0]
        self._token_sets(eng, sets)

    def _admit_packed(self, eng, group, first):
        """Prefill the (slot, request) pairs of one admission point: prompts longer than _PACKED_MAX_S one at a time
        (slot_prefill), all others in one slots_prefill. Each slot's first token goes to first[slot]. The packed
        prompts always fit the activations (max_batch * max_seq tokens): there are at most max_batch of them, each
        shorter than max_seq (_request)."""
        dev = first.device
        packed = []
        for s, r in group:
            if r.S > self._PACKED_MAX_S:
                feats = None if r.feats is None else r.feats.to(dev)
                vs = torch.tensor([r.vid_start], dtype=torch.int32, device=dev)
                eng.slot_prefill(s, r.ids.to(dev), feats, vs, tok_out=first[s:s + 1])
            else:
                packed.append((s, r))
        if packed:
            slots = [s for s, _ in packed]
            tok = eng.slots_prefill(slots, [r.ids for _, r in packed],
                                    [None if r.feats is None else r.feats.to(dev) for _, r in packed],
                                    [r.vid_start for _, r in packed])
            first[torch.tensor(slots, device=dev)] = tok

    def _prefill_chunked(self, eng, group, first, packed, sampling=False):
        """Prefill the (slot, request) pairs of one admission point whose prompts are longer than _PACKED_MAX_S on a
        paged engine: each prompt runs as consecutive chunks of _PACKED_MAX_S rows (Engine.slots_prefill_chunk),
        every chunk attending the columns its earlier chunks left in the slot's blocks. packed: chunk k of every
        prompt of the group goes into one call (at most n_slots * 512 rows, which the activations hold); otherwise
        each prompt runs alone. A slot's first token (first[slot]) is the one its last chunk gives. Returns the
        number of chunk calls. Every chunk call also draws a token for each of its prompts (only the last one's is
        kept), which a penalized slot adds to its token set: so the set is written again before each later call."""
        dev, L = first.device, self._PACKED_MAX_S
        calls = 0
        for batch in ([group] if packed else [[g] for g in group]):
            for start in range(0, max(r.S for _, r in batch), L):
                live = [(s, r) for s, r in batch if start < r.S]
                if sampling and start > 0:   # (chunk 0 follows the admission's write)
                    self._token_sets(eng, [(s, r.ids) for s, r in live if r.penalty != 1.0])
                tok = eng.slots_prefill_chunk([s for s, _ in live], [start] * len(live), [r.S for _, r in live],
                                              [r.ids[start:start + L] for _, r in live],
                                              [None if r.feats is None else r.feats.to(dev) for _, r in live],
                                              [r.vid_start for _, r in live])
                calls += 1
                for j, (s, r) in enumerate(live):
                    if start + L >= r.S:
                        first[s] = tok[j]
        return calls

    def _check_paged(self, reqs, chunked=False):
        """The requests a paged cache takes, checked on the host before any device work: a prompt of at most
        min(512, max_seq) tokens (a paged engine prefills packed) unless `chunked` (any prompt _request accepts), and
        at most kv_blocks - 1 blocks for the prompt and every new token, so that a request alone always fits the pool
        and the scheduler always makes progress."""
        C, usable = vn.KV_BLOCK_COLS, self._kv_blocks - 1
        s_lim = min(self._PACKED_MAX_S, self._max_seq)
        for i, r in enumerate(reqs):
            if r.start == 0 and r.S > s_lim and not chunked:
                raise ValueError(f"request {i}: prompt of {r.S} tokens; a paged KV cache takes prompts of at most "
                                 f"{s_lim} tokens (the packed prefill); chunked_prefill=True takes longer ones")
            need = -(-(r.S + r.n) // C)
            if need > usable and r.start > 0:
                raise ValueError(f"request {i}: conversation of {r.S} tokens + max_new_tokens {r.n} needs {need} blocks "
                                 f"of {C} columns, more than the pool's {usable} (kv_blocks {self._kv_blocks}, block 0 "
                                 "is the park block)")
            if need > usable:
                raise ValueError(f"request {i}: prompt {r.S} + max_new_tokens {r.n} needs {need} blocks of {C} columns, "
                                 f"more than the pool's {usable} (kv_blocks {self._kv_blocks}, block 0 is the park block)")

    def _schedule_paged(self, eng, reqs, n_slots, packed_admission, sampling, eos, chunked=False, lps=None):
        """The admission / decode loop of generate_requests on a paged KV cache. The host keeps a free list and each
        slot's row of the block table (block 0, the park block, wherever no request owns a block), and writes the
        whole table to the engine before every prefill and every decode chunk.
        - Blocks. A running request at position pos, decoding a chunk of m steps, owns the blocks of columns
          0 .. min(pos + m, S + n) - 1: every column the chunk writes that the request can still read (past S + n - 1
          the request has all its tokens; those columns of a chunk land in the park block or in its own last block).
        - Admission. Swapped-out requests resume first, oldest admission first, then queued requests in queue order
          (none overtakes another): each into a free slot when the free list covers its blocks for one chunk.
        - Preemption. When a chunk's growth is not covered, the most recently admitted running request is swapped out
          (its written blocks copied to pinned host memory, its blocks freed, its slot parked) until it is. Its
          position, pending token and sampling entry stay on the host; it resumes into any free slot and free blocks,
          restored exactly, and its tokens depend on its seed and positions only.
        - Chunked prefill (`chunked`). A prompt over _PACKED_MAX_S tokens is admitted by the same rule (its prompt's
          blocks plus one chunk's growth) and prefilled at its admission point by _prefill_chunked, before the next
          decode chunk; so a request that is swapped out always holds its whole prompt.
        - Sessions. A request with a "session" or "continues" key keeps its conversation when it ends (self._sessions):
          its tokens [L] and the blocks of columns 0 .. L - 2, which stay out of the free list, also across calls;
          its other blocks are freed. A continuation is admitted by the same rule with its conversation's blocks in
          its slot's row (copied back into fresh blocks first if they were swapped out) and prefills its tail, the
          columns L - 1 .. S - 1, through Engine.slots_prefill_append.
        - Eviction. Kept conversations are idle: when an admission, a resume or a chunk's growth is short of blocks,
          the least recently used one that is resident is swapped to pinned host memory (its blocks freed) before
          anything waits or any running request is preempted.
        - Log-probs (lps). A request swapped out before its first token reached the host takes that token's row
          along (it lives in its old slot's entry); every other row is read after the chunk that produced it.
        _check_paged guarantees that the oldest running request alone always fits."""
        dev, C, K = self.device, vn.KV_BLOCK_COLS, self._SLOT_CHUNK
        lps = lps or _RequestLogprobs(eng, reqs, n_slots, self.device)
        sessions = self._sessions
        table = [[0] * eng.table_row for _ in range(eng.n_slots)]    # every slot of the engine, parked
        kept = {b for ss in sessions.values() if ss.blocks is not None for b in ss.blocks}
        free = [b for b in range(eng.kv_blocks - 1, 0, -1) if b not in kept]   # pop() takes the lowest block
        results = [None] * len(reqs)
        queue = collections.deque(range(len(reqs)))
        owner = [None] * n_slots            # request of each slot
        pos = [0] * n_slots                 # tokens in each slot's cache; a slot without a request is parked at 0
        unseen = [False] * n_slots          # the slot's first token has not reached the host yet
        order = [0] * n_slots               # admission stamp of the slot's request (the latest is preempted first)
        blocks = [[] for _ in range(n_slots)]
        gen = {}
        swapped = {}                        # request -> (pos, pending token, unseen, host copies of its blocks)
        released = []                       # host buffers whose copy back may still be in flight
        stats = dict(preemptions=0, swapped_bytes=0, peak_blocks=0, kv_blocks=eng.kv_blocks, chunked_prefills=0,
                     chunk_calls=0, continuations=0, reused_rows=0, session_swaps=0, session_swapped_bytes=0)
        first = torch.zeros(n_slots, dtype=torch.int32, device=dev)     # the token each slot is fed next
        stamp = 0

        def cover(i, p, m):                 # blocks of columns 0 .. min(p + m, S + n) - 1
            r = reqs[i]
            return -(-min(p + m, r.S + r.n) // C)

        def take(s, want):
            while len(blocks[s]) < want:
                blocks[s].append(free.pop())
            table[s][:len(blocks[s])] = blocks[s]
            stats["peak_blocks"] = max(stats["peak_blocks"], eng.kv_blocks - 1 - len(free))

        def release(s, keep=0):             # the first `keep` blocks stay with a kept conversation
            free.extend(reversed(blocks[s][keep:]))
            blocks[s], table[s] = [], [0] * eng.table_row
            owner[s], pos[s] = None, 0

        def evict_session(spare=None):
            """swap the least recently used resident conversation (not `spare`) to host memory; False if none"""
            keys = [k for k, ss in sessions.items() if ss.blocks is not None and k != spare]
            if not keys:
                return False
            ss = sessions[min(keys, key=lambda k: sessions[k].used)]
            ss.saved = []
            for b in ss.blocks:
                buf = eng.swap_buffer()
                eng.kv_block_copy(b, buf)
                ss.saved.append(buf)
            free.extend(reversed(ss.blocks))
            ss.blocks = None
            stats["session_swaps"] += 1
            stats["session_swapped_bytes"] += len(ss.saved) * eng.block_bytes
            return True

        def swap_out(s):
            i = owner[s]
            if unseen[s]:
                lps.collect([(s, i, 1)])
            saved = []
            for b in blocks[s][:-(-pos[s] // C)]:        # the blocks that hold written columns
                buf = eng.swap_buffer()
                eng.kv_block_copy(b, buf)
                saved.append(buf)
            swapped[i] = (pos[s], int(first[s]), unseen[s], saved)
            stats["preemptions"] += 1
            stats["swapped_bytes"] += len(saved) * eng.block_bytes
            release(s)

        while True:
            idle = [s for s in range(n_slots) if owner[s] is None]
            admitted, resumed, tails = [], [], []
            while swapped and idle:
                i = min(swapped)            # requests are first admitted in queue (= index) order
                p, tok, uns, saved = swapped[i]
                while len(free) < cover(i, p, K) and evict_session():
                    pass
                if len(free) < cover(i, p, K):
                    break
                s = idle.pop(0)
                del swapped[i]
                stamp += 1
                owner[s], pos[s], unseen[s], order[s] = i, p, uns, stamp
                take(s, cover(i, p, K))
                for b, buf in zip(blocks[s], saved):
                    eng.kv_block_copy(b, buf, write=True)
                released.extend(saved)
                first[s] = tok
                resumed.append((s, i))
            while not swapped and idle and queue:
                i = queue[0]
                r = reqs[i]
                ss = sessions[r.continues] if r.continues is not None else None
                own = ss.blocks if ss is not None and ss.blocks is not None else []
                need = cover(i, r.S, K) - len(own)
                while len(free) < need and evict_session(spare=r.continues):
                    pass
                if len(free) < need:
                    break
                queue.popleft()
                s = idle.pop(0)
                stamp += 1
                owner[s], pos[s], unseen[s], order[s], gen[i] = i, r.S, True, stamp, []
                if ss is None:
                    take(s, cover(i, r.S, K))
                    admitted.append((s, i))
                    continue
                del sessions[r.continues]
                blocks[s] = list(own)
                take(s, cover(i, r.S, K))
                if ss.saved is not None:    # swapped out: copied back into the slot's first blocks
                    for b, buf in zip(blocks[s], ss.saved):
                        eng.kv_block_copy(b, buf, write=True)
                    released.extend(ss.saved)
                tails.append((s, i))
                stats["continuations"] += 1
                stats["reused_rows"] += r.start
            if admitted or resumed or tails:
                eng.set_block_table(table)
            if sampling and (admitted or resumed or tails):
                # a resumed request's token set: its prompt and its tokens, the pending one too when the host has
                # not seen it yet (its prefill's token)
                self._admit_sampling(eng, [(s, reqs[i]) for s, i in admitted + tails],
                                     [(s, reqs[i], gen[i] + ([int(first[s])] if unseen[s] else [])) for s, i in resumed])
            lps.sync(owner)
            # continuations: the tails admitted here in one call under packed_admission, one call each otherwise
            for group in ([tails] if packed_admission and tails else [[t] for t in tails]):
                tok = eng.slots_prefill_append([s for s, _ in group], [reqs[i].start for _, i in group],
                                               [reqs[i].ids[reqs[i].start:] for _, i in group])
                first[torch.tensor([s for s, _ in group], device=dev)] = tok
            if chunked and admitted:
                long = [(s, reqs[i]) for s, i in admitted if reqs[i].S > self._PACKED_MAX_S]
                admitted = [(s, i) for s, i in admitted if reqs[i].S <= self._PACKED_MAX_S]
                if long:
                    stats["chunked_prefills"] += len(long)
                    stats["chunk_calls"] += self._prefill_chunked(eng, long, first, packed_admission, sampling)
            if admitted and packed_admission:
                self._admit_packed(eng, [(s, reqs[i]) for s, i in admitted], first)
            elif admitted:
                for s, i in admitted:
                    r = reqs[i]
                    feats = None if r.feats is None else r.feats.to(dev)
                    vs = torch.tensor([r.vid_start], dtype=torch.int32, device=dev)
                    eng.slot_prefill(s, r.ids.to(dev), feats, vs, tok_out=first[s:s + 1])
            active = [s for s in range(n_slots) if owner[s] is not None]
            if not active:
                eng.set_block_table(table)      # every slot parked again
                stats["sessions"] = len(sessions)
                stats["sessions_resident"] = sum(ss.blocks is not None for ss in sessions.values())
                stats["sessions_swapped"] = stats["sessions"] - stats["sessions_resident"]
                self.last_kv_stats = stats
                return results
            m = min([K] + [self._max_seq - pos[s] for s in active])
            # growth, oldest admission first; while the free list falls short, swap out a kept conversation, else
            # preempt the latest running request
            for s in sorted(active, key=lambda t: order[t]):
                while owner[s] is not None and len(free) < cover(owner[s], pos[s], m) - len(blocks[s]):
                    if evict_session():
                        continue
                    swap_out(max((t for t in range(n_slots) if owner[t] is not None), key=lambda t: order[t]))
                if owner[s] is not None:
                    take(s, cover(owner[s], pos[s], m))
            active = [s for s in active if owner[s] is not None]
            eng.set_block_table(table)
            lps.sync(owner)
            out = eng.slot_decode(first, pos, m + 1)
            first = out[:, m].contiguous()
            host = out.tolist()
            released.clear()                # the stream has passed every copy enqueued before the decode
            running = [(s, owner[s]) for s in active]
            for s in active:
                i = owner[s]
                r = reqs[i]
                pos[s] += m
                for t in (host[s] if unseen[s] else host[s][1:]):
                    gen[i].append(t)
                    if self._request_done(r, gen[i], eos):
                        seq = torch.cat([r.ids, torch.tensor(gen[i], dtype=torch.int64)])
                        results[i] = seq[None].to(dev)
                        key = r.continues if r.continues is not None else r.session
                        keep = 0
                        if key is not None:     # kept: columns 0 .. L - 2, generate_continue's cache
                            keep = -(-(seq.numel() - 1) // C)
                            self._session_clock += 1
                            sessions[key] = SimpleNamespace(ids=seq, blocks=blocks[s][:keep], saved=None,
                                                            used=self._session_clock)
                        release(s, keep)
                        break
                unseen[s] = False
            lps.collect([(s, i, len(gen[i])) for s, i in running])

    def _request(self, i, r, max_new_tokens, stopping_criteria, n_vid, samp=None):
        """One request of generate_requests, checked on the host -> (ids [S] int64 on the host, S, n, feats,
        vid_start, criteria, and its sampling-table entry: temperature (0: greedy), top_k, seed)"""
        if isinstance(r, torch.Tensor):
            r = {"input_ids": r}
        ids = torch.as_tensor(r["input_ids"]).detach().cpu().to(torch.int64)
        if ids.dim() == 2 and ids.shape[0] == 1:
            ids = ids[0]
        if ids.dim() != 1 or ids.numel() == 0:
            raise ValueError(f"request {i}: input_ids must be [S] or [1, S], got shape {tuple(ids.shape)}")
        S, n = ids.numel(), int(r.get("max_new_tokens", max_new_tokens))
        if n < 1 or S + n > self._max_seq:
            raise ValueError(f"request {i}: prompt length {S} + max_new_tokens {n} does not fit max_seq {self._max_seq}")
        feats, vs = r.get("video_spatio_temporal_features"), vn.NO_VIDEO
        if feats is not None and r.get("continues") is not None:
            raise ValueError(f"request {i}: a continuation carries text only (its video is in the kept cache)")
        if feats is not None:
            if feats.dim() == 3 and feats.shape[0] == 1:
                feats = feats[0]
            if feats.dim() != 2 or feats.shape[0] != n_vid:
                raise ValueError(f"request {i}: video_spatio_temporal_features must be [{n_vid}, C], got "
                                 f"{tuple(feats.shape)}")
            vs = self._video_spans(ids[None], n_vid)[0]
        crit = r.get("stopping_criteria", stopping_criteria)
        samp = samp or dict(do_sample=False, temperature=1.0, top_k=50, seed=None)
        T, k, seed = 0.0, 0, 0
        top_p, penalty = self._nucleus_args(r.get("top_p", samp.get("top_p", 1.0)),
                                            r.get("repetition_penalty", samp.get("repetition_penalty", 1.0)),
                                            f"request {i}", r.get("do_sample", samp["do_sample"]))
        if r.get("do_sample", samp["do_sample"]):
            own = r.get("seed") is not None       # a seed is there (generate_requests checks it first)
            T, k, seed = self._sampling_args(r.get("temperature", samp["temperature"]), r.get("top_k", samp["top_k"]),
                                             r["seed"] if own else samp["seed"], f"request {i}")
            seed = seed if own else (seed + i) % 2 ** 64
            if T == 0:
                k, seed = 0, 0
        if T == 0:
            top_p = 1.0                           # HF adds no warpers when greedy
        return SimpleNamespace(ids=ids, S=S, n=n, feats=feats, vid_start=vs, criteria=list(crit or []),
                               temperature=T, top_k=k, seed=seed, top_p=top_p, penalty=penalty, session=r.get("session"),
                               continues=r.get("continues"), start=0, lp=r.get("logprobs", samp.get("logprobs")))

    def _bind_sessions(self, reqs):
        """The "session" / "continues" keys of generate_requests' requests, checked on the host before any device
        work. A continuation's ids become the whole conversation (the kept tokens, then its new turn), its S their
        length and its start the first column its tail prefill writes: the kept position L - 1, where
        generate_continue would start."""
        started, continued = {}, {}
        for i, r in enumerate(reqs):
            if r.session is not None and r.continues is not None:
                raise ValueError(f"request {i}: a request starts a conversation (\"session\") or continues one "
                                 "(\"continues\"), not both")
            if r.session is not None:
                if r.session in self._sessions:
                    raise ValueError(f"request {i}: a conversation is already kept under session key {r.session!r} "
                                     "(continue it, or end_session it first)")
                if r.session in started:
                    raise ValueError(f"request {i}: session key {r.session!r} is also started by request "
                                     f"{started[r.session]}")
                started[r.session] = i
            if r.continues is not None:
                if r.continues in continued:
                    raise ValueError(f"request {i}: conversation {r.continues!r} is also continued by request "
                                     f"{continued[r.continues]}; one turn per conversation and call")
                continued[r.continues] = i
        for key, i in continued.items():
            r = reqs[i]
            if key in started:
                raise ValueError(f"request {i}: conversation {key!r} is started by request {started[key]} in the same "
                                 "call; a turn's text depends on the previous answer, so continue it in a later call")
            if key not in self._sessions:
                raise ValueError(f"request {i}: no conversation is kept under key {key!r}")
            if r.S + 1 > self._PACKED_MAX_S:
                raise ValueError(f"request {i}: the continuation's tail (the last kept token and {r.S} new tokens) "
                                 f"has {r.S + 1} rows, more than {self._PACKED_MAX_S}")
            conv = self._sessions[key].ids
            L = conv.numel()
            if L + r.S + r.n > self._max_seq:
                raise ValueError(f"request {i}: conversation of {L} tokens + {r.S} new + max_new_tokens {r.n} does not "
                                 f"fit max_seq {self._max_seq}")
            r.ids, r.start = torch.cat([conv, r.ids]), L - 1
            r.S = r.ids.numel()

    def end_session(self, key=None):
        """Forget the conversation kept under `key` (every kept conversation when None): its cache blocks return to
        the free list of the next generate_requests call, and a copy swapped to host memory is dropped."""
        if key is None:
            self._sessions.clear()
            return
        if key not in self._sessions:
            raise ValueError(f"end_session: no conversation is kept under key {key!r}")
        del self._sessions[key]

    @staticmethod
    def _request_done(r, gen, eos):
        """Whether the request ends with its newest token gen[-1]: EOS, then the stopping criteria, then the
        length limit, in the order of _stepwise"""
        if eos is not None and gen[-1] == eos:
            return True
        if r.criteria:
            seq = torch.cat([r.ids, torch.tensor(gen, dtype=torch.int64)])[None]
            if any(c(seq, None) for c in r.criteria):
                return True
        return len(gen) >= r.n

    def generate_continue(self, new_input_ids, do_sample=False, temperature=1.0, max_new_tokens=32,
                          stopping_criteria=None, eos_token_id="config", pad_token_id=None, top_k=50, seed=None,
                          logprobs=None, top_p=1.0, repetition_penalty=1.0):
        """Next turn about the SAME video(s): `new_input_ids` [B, S_new] follow everything generated
        so far. Only the tokens the KV cache does not hold yet (the last generated token and the new
        text) are prefilled (vcl_llm_prefill_append); the reference re-runs the tower and the whole
        prompt every turn (chat.py:137-154). Returns the full sequence [B, S_total + n] like generate.
        After a left-padded generate the cache stays padded, so every row continues its own positions; the
        new text of every row has the same length S_new (no padding inside a turn).
        seed: do_sample=True samples on the device as generate(seed=...) does. logprobs: as in generate, for the new
        tokens of this turn. top_p / repetition_penalty: as in generate; the penalty's tokens are the whole
        conversation (every earlier turn, its answers as returned, and the new text)."""
        self._not_paged("generate_continue")
        if getattr(self, "_last_out", None) is None:
            raise ValueError("generate_continue: no previous generate() to continue")
        lp_n = self._logprobs_arg(logprobs, "generate_continue")
        if lp_n is not None and do_sample and seed is None:
            raise NotImplementedError("generate_continue: logprobs are computed by the device sampler, and sampling "
                                      "there needs seed= (unseeded do_sample=True draws from torch's RNG on the host)")
        self.last_logprobs = None
        top_p, penalty = self._nucleus_args(top_p, repetition_penalty, "generate_continue", do_sample,
                                            device=not do_sample or seed is not None)
        seeded = do_sample and seed is not None
        if seeded:
            temperature, top_k, seed = self._sampling_args(temperature, top_k, seed, "generate_continue")
        eng = self._ensure_engine(need_llm=True)
        prev = self._last_out
        tail = torch.cat([prev[:, self._pos:], new_input_ids.cuda().to(torch.int64)], dim=1)
        start = self._pos
        ctx = torch.cat([prev, new_input_ids.cuda().to(torch.int64)], dim=1)
        n = min(max_new_tokens, self._max_seq - ctx.shape[1])
        if n <= 0:
            raise ValueError(f"context length {ctx.shape[1]} leaves no room in max_seq {self._max_seq}")
        eos, pad = self._eos_pad(eos_token_id, pad_token_id)
        if seeded or lp_n is not None or (penalty != 1.0 and not do_sample):
            B, L = ctx.shape
            clips = list(range(B))
            if seeded:
                samp = self._sampling(eng, clips, [temperature] * B, [top_k] * B, [seed + b for b in clips], top_p,
                                      penalty)
            elif penalty != 1.0:   # greedy entries with the penalty
                samp = self._sampling(eng, clips, [0.0] * B, [0] * B, [0] * B, 1.0, penalty)
            else:
                samp = contextlib.nullcontext()
            if penalty != 1.0:
                self._token_sets(eng, [(b, ctx[b]) for b in clips])
            with samp, self._logprobs(eng, clips, lp_n):
                _, _, tok = eng.prefill_append(tail, start)
                first = eng.decode_loop(tok, ctx.shape[1], min(n, self._GREEDY_CHUNK))
                self._last_out = self._host_stops(eng, ctx, first, n, stopping_criteria, eos, pad)
            if lp_n is not None:   # the cache keeps the padding of the generate it continues
                pads = self._pads
                self.last_logprobs = self._read_logprobs(eng, self._last_out[:, L:].cpu(),
                                                         [L - (pads[b] if pads else 0) for b in range(B)], lp_n, eos)
            return self._last_out
        _, logits, _ = eng.prefill_append(tail, start, want_logits=True, want_token=False)
        self._pos = ctx.shape[1]
        self._last_out = self._stepwise(eng, ctx, logits, n, do_sample, temperature, stopping_criteria, eos, pad, top_k,
                                        top_p, penalty)
        return self._last_out

    @staticmethod
    def _host_processors(out, logits, sampled, temperature, top_k, top_p, penalty):
        """HF's logits processors of the stepwise path, in HF's order, on logits [B, V] fp32 after the ids `out`
        [B, L]: RepetitionPenaltyLogitsProcessor, then (sampled only) TemperatureLogitsWarper, TopKLogitsWarper and
        TopPLogitsWarper (min_tokens_to_keep 1); a dropped token is -inf"""
        if penalty != 1.0:
            ids = out.to(logits.device)
            sc = torch.gather(logits, 1, ids)
            sc = torch.where(sc < 0, sc * penalty, sc / penalty)
            logits = logits.scatter(1, ids, sc)
        if not sampled:
            return logits
        lg = logits / temperature
        if top_k and top_k < lg.shape[-1]:
            kth = torch.topk(lg, top_k, dim=-1).values[:, -1:]
            lg = lg.masked_fill(lg < kth, float("-inf"))
        if top_p < 1.0:
            srt, idx = torch.sort(lg, descending=False)
            drop = srt.softmax(dim=-1).cumsum(dim=-1) <= (1 - top_p)
            drop[..., -1:] = False
            lg = lg.masked_fill(drop.scatter(1, idx, drop), float("-inf"))
        return lg

    def _stepwise(self, eng, out, logits, n, do_sample, temperature, stopping_criteria, eos, pad, top_k=50, top_p=1.0,
                  penalty=1.0):
        """One token per C-ABI call. After the loop the cache holds every returned token but the last
        (self._pos = out.shape[1] - 1), the state generate_continue starts from. The logits go through HF's
        processors in HF's order: repetition penalty (over `out` so far), then temperature, top-k and top-p."""
        unfinished = torch.ones(out.shape[0], dtype=torch.bool, device=out.device)
        for step in range(n):
            lg = self._host_processors(out, logits, do_sample and temperature > 0, temperature, top_k, top_p, penalty)
            if do_sample and temperature > 0:
                nxt = torch.multinomial(torch.softmax(lg, dim=-1), 1)[:, 0]
            else:
                nxt = lg.argmax(-1)
            if eos is not None:
                nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad))
            out = torch.cat([out, nxt[:, None].to(torch.int64)], dim=1)
            if eos is not None:
                unfinished = unfinished & (nxt != eos)
                if not bool(unfinished.any()):
                    break
            if stopping_criteria and any(c(out, None) for c in stopping_criteria):
                break
            if step + 1 == n or self._pos >= self._max_seq:
                break
            logits, _ = eng.decode_step(nxt.to(torch.int32).contiguous(), self._pos, want_logits=True)
            self._pos += 1
        return out


class _RequestLogprobs:
    """The log-probs of one generate_requests call: the slots' entries as the engine holds them, and each request's
    rows read so far (blocks of rows, one row per new token, in order). Request i's k-th new token took position
    reqs[i].S + k of its slot's entry."""

    def __init__(self, eng, reqs, n_slots, dev):
        self.eng, self.reqs, self.dev = eng, reqs, dev
        self.on = any(r.lp is not None for r in reqs)
        self.written = [-1] * n_slots
        self.rows = {i: [] for i, r in enumerate(reqs) if r.lp is not None}
        self.have = {i: 0 for i in self.rows}

    def sync(self, owner):
        """One set_logprobs call for the slots whose entry changed: the top_n of the slot's request, -1 without one"""
        if not self.on:
            return
        want = [-1 if i is None or self.reqs[i].lp is None else self.reqs[i].lp for i in owner]
        changed = [s for s, w in enumerate(want) if w != self.written[s]]
        if changed:
            self.eng.set_logprobs(changed, [want[s] for s in changed])
            for s in changed:
                self.written[s] = want[s]

    def collect(self, running):
        """(slot, request, its new tokens so far): read the rows the host does not hold yet, all in one copy"""
        reads = [(s, i, self.have[i], n - self.have[i]) for s, i, n in running if i in self.rows and n > self.have[i]]
        if not reads:
            return
        total = sum(c for *_, c in reads)
        ids = torch.empty(total, vn.LOGPROB_PLACES, dtype=torch.int32, device=self.dev)
        lp = torch.empty(total, vn.LOGPROB_PLACES, dtype=torch.float32, device=self.dev)
        o = 0
        for s, i, had, c in reads:
            self.eng.read_logprobs(s, self.reqs[i].S + had, c, ids_out=ids[o:o + c], lp_out=lp[o:o + c])
            o += c
        ids, lp = ids.cpu(), lp.cpu()
        o = 0
        for s, i, had, c in reads:
            self.rows[i].append((ids[o:o + c], lp[o:o + c]))
            self.have[i] += c
            o += c

    def result(self):
        out = [None] * len(self.reqs)
        for i, rows in self.rows.items():
            ids = torch.cat([a for a, _ in rows])
            lp = torch.cat([b for _, b in rows])
            out[i] = VideoChatGPTLlamaForCausalLM._logprob_entry(ids, lp, self.reqs[i].lp)
        return out

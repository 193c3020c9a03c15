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

import contextlib
import json
import math
import numbers
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
from . import inflight  # noqa: E402
from . import candidates as candidate_scoring  # noqa: E402
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


class _BeamReplay:
    """Steps 4-6 of transformers' _beam_search (generation/utils.py, do_sample=False) replayed in fp32 torch on the
    host, one step per device record, for B prompts of k beams, prompt length S (with its left padding, HF's
    decoder_prompt_len) and n new tokens at most (max_length = S + n). Per step t (cur_len = S + t) it takes the K = 2k
    candidates (score, parent beam, token), best first, and the device's k running picks:
      hit       token == eos, or cur_len + 1 >= max_length
      finished  the hits among the first k candidates, score / (cur_len + 1 - S) ** length_penalty, with -1e9 added
                when the item's k finished slots are full and early_stopping is True, when the early-stop heuristic
                is satisfied, and to every candidate that did not just finish; merged with the kept finished set by
                top k
      running   the picked candidates, with score + hit * -1e9
      heuristic HF's _check_early_stop_heuristic, and the call ends when no item can improve, or (early_stopping
                True) every finished set is full, or every candidate hit.
    Sequences are the generated tokens only, filled with (pad or eos) when eos is set, else -1, as HF fills them."""

    def __init__(self, B, k, S, n, eos, pad, length_penalty, early_stopping):
        self.B, self.k, self.S, self.n = B, k, S, n
        self.eos, self.lp, self.early = eos, float(length_penalty), early_stopping
        self.max_length = S + n
        fill = (pad if pad else eos) if eos is not None else -1
        self.run_seq = torch.full((B, k, n), fill, dtype=torch.int64)
        self.fin_seq = torch.full((B, k, n), fill, dtype=torch.int64)
        self.fin_score = torch.full((B, k), -1.0e9, dtype=torch.float32)
        self.fin_len = torch.zeros((B, k), dtype=torch.int64)          # generated tokens of a finished hypothesis
        self.is_fin = torch.zeros((B, k), dtype=torch.bool)
        self.unsat = torch.ones((B, 1), dtype=torch.bool)              # the early-stop heuristic is unsatisfied
        self.first_k = torch.arange(2 * k) < k
        self.t = 0                                                      # steps replayed

    @staticmethod
    def _take(x, idx):
        """x [B, M, ...] gathered along dim 1 by idx [B, N]"""
        while idx.dim() < x.dim():
            idx = idx.unsqueeze(-1)
        return torch.take_along_dim(x, idx, dim=1)

    def step(self, score, beam, tok, pick):
        """One step: score f32 [B, K], beam / tok int64 [B, K], pick int64 [B, k]. Returns True when HF stops."""
        t, S = self.t, self.S
        cur_len = S + t
        cand_seq = self._take(self.run_seq, beam).clone()
        cand_seq[:, :, t] = tok
        hit = torch.full_like(tok, cur_len + 1 >= self.max_length, dtype=torch.bool)
        if self.eos is not None:
            hit = hit | (tok == self.eos)
        # finished hypotheses
        just = hit & self.first_k[None, :]
        fin = score / ((cur_len + 1 - S) ** self.lp)
        full = torch.all(self.is_fin, dim=-1, keepdim=True) & (self.early is True)
        fin = fin + full.to(torch.float32) * -1.0e9
        fin = fin + (~self.unsat).to(torch.float32) * -1.0e9
        fin = fin + (~just).to(torch.float32) * -1.0e9
        merged = torch.cat([self.fin_score, fin], dim=1)
        keep = torch.topk(merged, k=self.k, dim=1)[1]
        self.fin_seq = self._take(torch.cat([self.fin_seq, cand_seq], dim=1), keep)
        self.fin_score = self._take(merged, keep)
        self.fin_len = self._take(torch.cat([self.fin_len, torch.full_like(tok, t + 1)], dim=1), keep)
        self.is_fin = self._take(torch.cat([self.is_fin, just], dim=1), keep)
        # running beams: the device's picks
        run_score = self._take(score + hit.to(torch.float32) * -1.0e9, pick)
        self.run_seq = self._take(cand_seq, pick)
        self.t = t + 1
        cur_len += 1
        # early stopping
        if self.early == "never" and self.lp > 0.0:
            best_len = self.max_length - S
        else:
            best_len = cur_len - S
        best = run_score[:, :1] / (best_len ** self.lp)
        worst = torch.where(self.is_fin, torch.min(self.fin_score, dim=1, keepdim=True)[0], -1.0e9)
        self.unsat = self.unsat & torch.any(best > worst, dim=-1, keepdim=True)
        improvable = bool(self.unsat.any())
        open_beam = not (bool(self.is_fin.all()) and self.early is True)
        return not (improvable and open_beam and not bool(hit.all()))

    def steps(self, rec, picks):
        """The records [n, B, K, 3] and picks [n, B, k] of a chunk, step by step; True once HF stops (later steps of
        the chunk are discarded)"""
        rec, picks = rec.cpu(), picks.cpu().to(torch.int64)
        score, beam, tok = vn.beam_records(rec)
        for i in range(rec.shape[0]):
            if self.step(score[i], beam[i], tok[i], picks[i]):
                return True
        return False

    def result(self, m):
        """(sequences int64 [B * m, longest], sequences_scores f32 [B * m]): each prompt's m best finished
        hypotheses, best first, cut at the longest of them"""
        length = int(self.fin_len[:, :m].max())
        seqs = self.fin_seq[:, :m].reshape(self.B * m, self.n)[:, :length]
        return seqs, self.fin_score[:, :m].reshape(-1).clone()


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
        self.last_beam_scores = None   # generate(num_beams > 1): HF's sequences_scores, f32 [B * num_return_sequences]
        self._after_beams = False      # the last generate ran beam search: there is no single turn to continue
        self._after_contrastive = False   # ... or contrastive search (generate_continue refuses both)
        self._pads = None              # the left padding of the last generate (log-prob positions of generate_continue)
        self._sessions: dict = {}      # kept conversations of generate_requests (paged): key -> inflight.PagedSlots' state
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

    def _spans_dev(self, ids, feats, n_vid, n_pad=None, device="cuda"):
        starts = self._video_spans(ids, n_vid, n_pad) if feats is not None else [vn.NO_VIDEO] * ids.shape[0]
        return torch.tensor(starts, dtype=torch.int32, device=device)

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

    def _warper_args(self, min_p, typical_p, epsilon_cutoff, eta_cutoff, what="generate", sampled=True, device=True):
        """Checks HF's min-p / typical / epsilon / eta settings on the host, with HF's messages -> None when the call
        runs none of them (greedy calls ignore them, as HF adds no warpers there), else (min_p, typical_p, epsilon,
        eta) as floats with off as 0, 1, 0, 0. On as in HF's _get_logits_processor: min_p not None, typical_p < 1,
        0 < epsilon_cutoff < 1, 0 < eta_cutoff < 1. The device sampler's vocabulary limit applies when the call runs
        there (`device`)."""
        mp = 0.0 if min_p is None else float(min_p)
        if not 0.0 <= mp <= 1.0:
            raise ValueError(f"{what}: `min_p` has to be a float in the [0, 1] interval, but is {min_p}")
        ty = 1.0 if typical_p is None else float(typical_p)
        if ty < 1.0 and not ty > 0.0:
            raise ValueError(f"{what}: `typical_p` has to be a float > 0 and < 1, but is {typical_p}")
        ty = ty if ty < 1.0 else 1.0
        ep = 0.0 if epsilon_cutoff is None else float(epsilon_cutoff)
        ep = ep if 0.0 < ep < 1.0 else 0.0
        et = 0.0 if eta_cutoff is None else float(eta_cutoff)
        et = et if 0.0 < et < 1.0 else 0.0
        if not sampled or (mp == 0.0 and ty == 1.0 and ep == 0.0 and et == 0.0):   # (min_p 0 removes nothing)
            return None
        V = self.config.vocab_size
        if device and V > vn.SAMPLE_WIDE_MAX_V:
            raise ValueError(f"{what}: min_p, typical_p, epsilon_cutoff and eta_cutoff take a vocabulary of at most "
                             f"{vn.SAMPLE_WIDE_MAX_V} tokens on the device sampler, this model has {V}")
        return mp, ty, ep, et

    @staticmethod
    def _set_entries(eng, clips, temperature, top_k, seeds, top_p, penalty, warpers=None):
        """One sampling-table write: set_sampling when every entry has top_p 1 and penalty 1 (what a call without
        them always made), set_sampling_ex otherwise; then, when some entry of `warpers` (each None or
        _warper_args' tuple) is on, set_warpers for every entry"""
        if all(p == 1.0 for p in top_p) and all(r == 1.0 for r in penalty):
            eng.set_sampling(clips, temperature, top_k, seeds)
        else:
            eng.set_sampling_ex(clips, temperature, top_k, seeds, top_p, penalty)
        if warpers is not None and any(w is not None for w in warpers):
            cols = list(zip(*[w if w is not None else (0.0, 1.0, 0.0, 0.0) for w in warpers]))
            eng.set_warpers(clips, *cols)

    @contextlib.contextmanager
    def _sampling(self, eng, clips, temperature, top_k, seeds, top_p=1.0, penalty=1.0, warpers=None):
        """Entries `clips` of the engine's sampling table sample (temperature 0: greedy, with the penalty) for the
        duration of the block and are greedy, without top-p, penalty or warpers, again afterwards, also when the block
        raises."""
        n = len(clips)
        self._set_entries(eng, clips, temperature, top_k, seeds, [top_p] * n, [penalty] * n, [warpers] * n)
        try:
            yield
        finally:
            eng.set_sampling(clips, [0.0] * n, [0] * n, [0] * n)

    @staticmethod
    def _token_sets(eng, rows):
        """(entry, ids) pairs: each entry's token set of the repetition penalty becomes its ids, one call each"""
        for b, ids in rows:
            eng.set_token_set(b, ids)

    def _ban_args(self, no_repeat_ngram_size, bad_words_ids, min_new_tokens, eos, what="generate", device=True):
        """Checks the banned-token settings on the host, with HF's messages -> None when none is on, else
        SimpleNamespace(ngram (0: off), words (the bad words as HF keeps them: [eos] dropped, duplicates once; None when
        bad_words_ids is None), min_new (0 when off or EOS is disabled), eos). HF adds each processor when: n-gram size > 0,
        bad_words_ids given, min_new_tokens > 0 with an EOS."""
        n = 0 if no_repeat_ngram_size is None else no_repeat_ngram_size
        if isinstance(n, bool) or not isinstance(n, int) or n < 0:
            raise ValueError(f"{what}: `ngram_size` has to be a strictly positive integer, but is {n}")
        m = 0 if min_new_tokens is None else min_new_tokens
        if isinstance(m, bool) or not isinstance(m, int) or m < 0:
            raise ValueError(f"{what}: `min_new_tokens` has to be a positive integer, but is {m}")
        words = None
        if bad_words_ids is not None:
            b = bad_words_ids
            if not isinstance(b, list) or len(b) == 0:
                raise ValueError(f"{what}: `bad_words_ids` has to be a non-empty list, but is {b}.")
            if any(not isinstance(w, list) for w in b):
                raise ValueError(f"{what}: `bad_words_ids` has to be a list of lists, but is {b}.")
            if any(any(isinstance(t, bool) or not isinstance(t, numbers.Integral) or t < 0 for t in w) for w in b):
                raise ValueError(f"{what}: Each list in `bad_words_ids` has to be a list of positive integers, but is "
                                 f"{b}.")
            if any(len(w) == 0 for w in b):
                raise ValueError(f"{what}: Each list in `bad_words_ids` has to be a non-empty list of token ids, but "
                                 f"is {b}.")
            keep = {}                              # HF: {tuple(word): -inf} without [eos], in order
            for w in b:
                if eos is None or list(w) != [eos]:
                    keep.setdefault(tuple(int(t) for t in w), None)
            V = self.config.vocab_size
            bad = [t for w in keep for t in w if t >= V]
            if bad:
                raise ValueError(f"{what}: The model vocabulary size is {V}, but the following tokens were being "
                                 f"biased: {bad}")
            words = [list(w) for w in keep]
            size = sum(1 + len(w) for w in words)
            if size > vn.BAN_WORDS_MAX:
                raise ValueError(f"{what}: bad_words_ids take {size} int32 on the device (a length and the ids of each "
                                 f"word), more than {vn.BAN_WORDS_MAX}")
        if eos is None:
            m = 0                                  # HF adds no MinNewTokensLengthLogitsProcessor without an EOS
        if n == 0 and words is None and m == 0:
            return None
        V = self.config.vocab_size
        if device and V > vn.SAMPLE_WIDE_MAX_V:
            raise ValueError(f"{what}: no_repeat_ngram_size, bad_words_ids and min_new_tokens take a vocabulary of at "
                             f"most {vn.SAMPLE_WIDE_MAX_V} tokens on the device sampler, this model has {V}")
        return SimpleNamespace(ngram=n, words=words, min_new=m, eos=eos)

    @staticmethod
    def _set_bans(eng, clips, bans, eos, eos_from):
        """One ban-table write: clip clips[i] bans by bans[i] (None: off), EOS before column eos_from[i]"""
        eng.set_bans(clips, [b.ngram if b else 0 for b in bans],
                     [eos if b and b.min_new else -1 for b in bans], [e if b else 0 for b, e in zip(bans, eos_from)],
                     [b.words or [] if b else [] for b in bans])

    @contextlib.contextmanager
    def _banning(self, eng, clips, bans, eos, eos_from):
        """Entries `clips` ban by `bans` (None: nothing changes) for the duration of the block and are off again
        afterwards, also when the block raises"""
        if bans is None:
            yield
            return
        n = len(clips)
        self._set_bans(eng, clips, [bans] * n, eos, [eos_from] * n)
        try:
            yield
        finally:
            self._set_bans(eng, clips, [None] * n, eos, [0] * n)

    @staticmethod
    def _histories(eng, rows):
        """(entry, ids) pairs: each entry's token history becomes its ids, one call each"""
        for b, ids in rows:
            eng.set_token_history(b, ids)

    @staticmethod
    def _host_bans(out, logits, bans, S):
        """HF's NoRepeatNGramLogitsProcessor, NoBadWordsLogitsProcessor and MinNewTokensLengthLogitsProcessor, in that
        order, on logits [B, V] fp32 after the ids `out` [B, c] of a call whose first new token took column S (each
        as HF computes it: the n-gram and EOS bans assign -inf, the bad words add a bias of 0 / -inf)"""
        c = out.shape[1]
        rows = out.tolist()
        if bans.ngram:
            n = bans.ngram
            logits = logits.clone()
            if c + 1 >= n:
                for b, h in enumerate(rows):
                    key = h[c - n + 1:c]
                    banned = [h[i + n - 1] for i in range(c - n + 1) if h[i:i + n - 1] == key]
                    logits[b, banned] = float("-inf")
        if bans.words is not None:
            bias = torch.zeros_like(logits)
            for w in bans.words:
                if len(w) == 1:
                    bias[:, w[0]] = float("-inf")
            for w in bans.words:
                if 1 < len(w) <= c:
                    for b, h in enumerate(rows):
                        if h[c - len(w) + 1:] == w[:-1]:
                            bias[b, w[-1]] += float("-inf")
            logits = logits + bias
        if bans.min_new and c - S < bans.min_new:
            logits = logits.clone()
            logits[:, bans.eos] = float("-inf")
        return logits

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

    def _guidance_args(self, guidance_scale, neg_ids, neg_mask, neg_feats, input_ids, num_beams):
        """Checks the classifier-free guidance settings of generate on the host -> None (off: guidance_scale None or
        1.0, as HF adds no processor then) or the scale as a float"""
        if guidance_scale is None:
            return None
        g = float(guidance_scale)
        if not math.isfinite(g):
            raise ValueError(f"generate: guidance_scale {guidance_scale} must be a finite value (None or 1.0: off)")
        if g == 1.0:
            return None
        if not (isinstance(num_beams, int) and num_beams == 1):
            raise NotImplementedError(f"generate: guidance_scale is not supported with num_beams={num_beams!r}")
        B = input_ids.shape[0]
        if 2 * B > self._max_batch:
            raise ValueError(f"generate: guidance_scale with {B} prompts needs {2 * B} cache clips (every negative "
                             f"prompt takes one), more than max_batch {self._max_batch}")
        V = self.config.vocab_size
        if V > vn.SAMPLE_WIDE_MAX_V:
            raise ValueError(f"generate: guidance_scale takes a vocabulary of at most {vn.SAMPLE_WIDE_MAX_V} tokens on "
                             f"the device, this model has {V}")
        if neg_ids is not None and (neg_ids.dim() != 2 or neg_ids.shape[0] != B or neg_ids.shape[1] < 1):
            raise ValueError(f"generate: negative_prompt_ids {tuple(neg_ids.shape)} must be [B, S_neg] with B = {B}")
        if neg_mask is not None:
            if neg_ids is None:
                raise ValueError("generate: negative_prompt_attention_mask needs negative_prompt_ids")
            if tuple(neg_mask.shape) != tuple(neg_ids.shape):
                raise ValueError(f"generate: negative_prompt_attention_mask {tuple(neg_mask.shape)} does not match "
                                 f"negative_prompt_ids {tuple(neg_ids.shape)}")
        if neg_feats is not None:
            if neg_ids is None:
                raise ValueError("generate: negative_video_spatio_temporal_features needs negative_prompt_ids with a "
                                 "video span")
            if neg_feats.dim() != 3 or neg_feats.shape[0] != B:
                raise ValueError(f"generate: negative_video_spatio_temporal_features {tuple(neg_feats.shape)} must be "
                                 f"[B, tokens, channels] with B = {B}, one row per negative prompt")
        return g

    def _guided_batch(self, ids, pads, feats, neg_ids, neg_mask, neg_feats, n_vid):
        """The 2B rows of a guided prefill: the B prompts, then the B negative prompts (HF's default without one:
        each prompt's last token alone), all left-padded to the longest, each negative row with its own video span
        (negative features) or none. -> (ids2 [2B, S2], pads2 (None when nothing is padded), spans [2B], feats
        [2B, ., .] or None, shift = S2 - S). The prompts keep their tokens; the shift extra columns in front of a
        prompt repeat its first token and are padding."""
        B, S = ids.shape
        neg = ids[:, -1:] if neg_ids is None else neg_ids.to(ids.device, torch.int64)
        Sn = neg.shape[1]
        npad = left_padding(neg_mask, (B, Sn)) if neg_mask is not None else None
        S2 = max(S, Sn)
        shift = S2 - S
        cond = torch.cat([ids[:, :1].expand(B, shift), ids], dim=1)
        negp = torch.cat([neg[:, :1].expand(B, S2 - Sn), neg], dim=1)
        ids2 = torch.cat([cond, negp], dim=0).contiguous()
        pads2 = [shift + (pads[b] if pads else 0) for b in range(B)] + \
                [S2 - Sn + (npad[b] if npad else 0) for b in range(B)]
        cs = self._video_spans(cond, n_vid, pads2[:B]) if feats is not None else [vn.NO_VIDEO] * B
        ns = self._video_spans(negp, n_vid, pads2[B:]) if neg_feats is not None else [vn.NO_VIDEO] * B
        f2 = None
        if feats is not None or neg_feats is not None:
            like = feats if feats is not None else neg_feats
            zero = torch.zeros(B, *like.shape[1:], dtype=torch.bfloat16, device="cuda")
            f2 = torch.cat([zero if f is None else f.cuda().to(torch.bfloat16) for f in (feats, neg_feats)], dim=0)
        spans = torch.tensor(cs + ns, dtype=torch.int32, device=ids.device)
        return ids2, (pads2 if any(pads2) else None), spans, f2, shift

    @staticmethod
    def _host_guidance(cond, uncond, g):
        """HF's UnbatchedClassifierFreeGuidanceLogitsProcessor on fp32 logits [B, V] of the prompts and of their
        negative prompts: g * (log_softmax(cond) - log_softmax(uncond)) + log_softmax(uncond)"""
        lc = torch.log_softmax(cond.float(), dim=-1)
        lu = torch.log_softmax(uncond.float(), dim=-1)
        return g * (lc - lu) + lu

    @contextlib.contextmanager
    def _guiding(self, eng, B, g):
        """Clips 0 .. B-1 are guided by clips B .. 2B-1 with scale g (None: nothing changes) for the duration of the
        block, and the guidance table is off again afterwards, also when the block raises"""
        if g is None:
            yield
            return
        clips = list(range(2 * B))
        eng.set_guidance(clips, [B + b for b in range(B)] + [-1] * B, [g] * B + [1.0] * B)
        try:
            yield
        finally:
            eng.set_guidance(clips, [-1] * (2 * B), [1.0] * (2 * B))

    @torch.no_grad()
    def generate(self, input_ids, video_spatio_temporal_features=None, do_sample=False, temperature=1.0,
                 max_new_tokens=32, stopping_criteria=None, eos_token_id="config", pad_token_id=None, top_k=50,
                 attention_mask=None, seed=None, logprobs=None, top_p=1.0, repetition_penalty=1.0, num_beams=1,
                 num_return_sequences=1, length_penalty=1.0, early_stopping=False, no_repeat_ngram_size=None,
                 bad_words_ids=None, min_new_tokens=None, guidance_scale=None, negative_prompt_ids=None,
                 negative_prompt_attention_mask=None, negative_video_spatio_temporal_features=None, penalty_alpha=None,
                 min_p=None, typical_p=None, epsilon_cutoff=None, eta_cutoff=None, **kw):
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
        device loops with greedy entries; unseeded sampling applies them on the host, step by step, as HF does.
        no_repeat_ngram_size (None or 0: off), bad_words_ids (None: off) and min_new_tokens (None or 0: off): HF's
        NoRepeatNGramLogitsProcessor, NoBadWordsLogitsProcessor and MinNewTokensLengthLogitsProcessor, checked with
        HF's messages. They set the logits of banned tokens to -inf after the penalty, over the row's input_ids so far
        (padding and prompt included); min_new_tokens bans EOS until that many new tokens are out (nothing without
        an EOS). Seeded sampling and greedy calls apply them on the device (DESIGN.md section 3, "Banned tokens");
        unseeded sampling on the host, step by step.
        num_beams > 1: HF's beam search (do_sample=False), with HF's num_return_sequences, length_penalty and
        early_stopping (True, False or "never"); see _beam_generate. It returns [B * num_return_sequences, S + m], the
        best hypotheses of each prompt first, and sets self.last_beam_scores (HF's sequences_scores). Sampling, seed,
        logprobs, top_p, repetition_penalty, the banned-token settings and stopping criteria are not supported with
        beams (NotImplementedError), and
        a beam call must fit max_seq whole (S + max_new_tokens <= max_seq: a shorter call would move HF's max-length
        step and so change the search). num_beams must be an int 1 .. 8 on every call (a ValueError otherwise, rather
        than a silently greedy call); num_return_sequences without beams is ignored, as it always was.
        guidance_scale (None or 1.0: off): HF's classifier-free guidance (UnbatchedClassifierFreeGuidanceLogitsProcessor;
        DESIGN.md section 3). Every prompt is decoded next to an unconditional sequence, its negative prompt
        (negative_prompt_ids [B, S_neg], left-padded by negative_prompt_attention_mask; HF's default without one is the
        prompt's last token alone), which takes a cache clip of its own (2B <= max_batch), and the scores become
        g * (log_softmax(cond) - log_softmax(uncond)) + log_softmax(uncond) before every other processor. Each negative
        row runs as if alone (its positions start at its first real token). negative_video_spatio_temporal_features
        [B, ., .]: the pooled features of a video span in the negative prompts (e.g. a noised copy); without them a
        span is embedded as text, as generate does without features. Greedy and seeded calls guide on the device,
        unseeded sampling on the host step by step. Not with beams (NotImplementedError).
        penalty_alpha (None or 0: off) with top_k > 1: HF's contrastive search (DESIGN.md section 3, "Contrastive
        search"); see _contrastive_generate. Each step decodes the top_k most probable tokens of every prompt as cache
        clips of their own (B * top_k <= max_batch, a ValueError otherwise) and keeps the one that best trades its
        probability against its largest cosine similarity to the prompt's hidden states so far. It runs with
        attention_mask, EOS / pad_token_id, stopping criteria and video features; sampling, seed, beams, guidance,
        logprobs, top_p, repetition_penalty and the banned-token settings raise NotImplementedError. top_k <= 1
        decodes greedily, as in HF. generate_continue cannot continue it (ValueError).
        min_p (None: off), typical_p (None or >= 1: off), epsilon_cutoff and eta_cutoff (on when in (0, 1)): HF's
        MinPLogitsWarper, TypicalLogitsWarper, EpsilonLogitsWarper and EtaLogitsWarper, after top-p and in that order,
        when sampling (a greedy call ignores them, as HF does), checked with HF's messages. Seeded sampling applies them
        on the device (DESIGN.md section 3, "Min-p, typical, epsilon and eta"), guided calls after the guidance;
        unseeded sampling on the host, step by step. Not with beams or penalty_alpha (NotImplementedError)."""
        self._not_paged("generate")
        beams = not (isinstance(num_beams, int) and num_beams == 1)
        contrastive = penalty_alpha is not None and penalty_alpha != 0 and isinstance(top_k, int) and top_k > 1
        # on as _warper_args has it, so HF's off values (GenerationConfig's typical_p 1.0, epsilon / eta 0.0) pass
        warp_on = (beams or contrastive) and \
            self._warper_args(min_p, typical_p, epsilon_cutoff, eta_cutoff, "generate", device=False)
        if warp_on:
            name = next(n for n, v, off in zip(("min_p", "typical_p", "epsilon_cutoff", "eta_cutoff"), warp_on,
                                               (0.0, 1.0, 0.0, 0.0)) if v != off)
            raise NotImplementedError(f"generate: {name} is not supported with "
                                      f"{'num_beams > 1' if beams else 'penalty_alpha'} (both decode without "
                                      "sampling warpers)")
        cs = self._contrastive_args(penalty_alpha, top_k, do_sample, seed, num_beams, guidance_scale, logprobs, top_p,
                                    repetition_penalty, (no_repeat_ngram_size, bad_words_ids, min_new_tokens))
        if cs is not None:
            return self._contrastive_generate(input_ids, video_spatio_temporal_features, attention_mask, max_new_tokens,
                                              stopping_criteria, eos_token_id, pad_token_id, *cs)
        self._after_contrastive = False
        guide = self._guidance_args(guidance_scale, negative_prompt_ids, negative_prompt_attention_mask,
                                    negative_video_spatio_temporal_features, input_ids, num_beams)
        beams = self._beam_args(num_beams, num_return_sequences, length_penalty, early_stopping, do_sample, seed,
                                logprobs, top_p, repetition_penalty, stopping_criteria,
                                (no_repeat_ngram_size, bad_words_ids, min_new_tokens))
        if beams is not None:
            return self._beam_generate(input_ids, video_spatio_temporal_features, attention_mask, max_new_tokens,
                                       eos_token_id, pad_token_id, *beams)
        self._after_beams, self.last_beam_scores = False, None
        lp_n = self._logprobs_arg(logprobs, "generate")
        if lp_n is not None and do_sample and seed is None:
            raise NotImplementedError("generate: logprobs are computed by the device sampler, and sampling there needs "
                                      "seed= (unseeded do_sample=True draws from torch's RNG on the host)")
        top_p, penalty = self._nucleus_args(top_p, repetition_penalty, "generate", do_sample,
                                            device=not do_sample or seed is not None)
        warp = self._warper_args(min_p, typical_p, epsilon_cutoff, eta_cutoff, "generate", do_sample and
                                 float(temperature) > 0, device=seed is not None)
        eos, pad = self._eos_pad(eos_token_id, pad_token_id)
        bans = self._ban_args(no_repeat_ngram_size, bad_words_ids, min_new_tokens, eos, "generate",
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
        self._pads = pads
        self._shift = 0
        if guide is not None:
            return self._guided_generate(eng, ids, pads, feats, negative_prompt_ids, negative_prompt_attention_mask,
                                         negative_video_spatio_temporal_features, guide, max_new_tokens, do_sample,
                                         seeded, temperature, top_k, seed, top_p, penalty, bans, lp_n,
                                         stopping_criteria, eos, pad, warp)
        if seeded or lp_n is not None or ((penalty != 1.0 or bans) and not do_sample):
            clips = list(range(B))
            if seeded:
                samp = self._sampling(eng, clips, [temperature] * B, [top_k] * B, [seed + b for b in clips], top_p,
                                      penalty, warp)
            elif penalty != 1.0:   # greedy entries with the penalty
                samp = self._sampling(eng, clips, [0.0] * B, [0] * B, [0] * B, 1.0, penalty)
            else:
                samp = contextlib.nullcontext()
            if penalty != 1.0:
                self._token_sets(eng, [(b, ids[b]) for b in clips])
            if bans:
                self._histories(eng, [(b, ids[b]) for b in clips])
            with samp, self._banning(eng, clips, bans, eos, S + (bans.min_new if bans else 0)), \
                    self._logprobs(eng, clips, lp_n):
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
                                            top_k, top_p, penalty, bans, warpers=warp)
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

    def _guided_generate(self, eng, ids, pads, feats, neg_ids, neg_mask, neg_feats, g, max_new_tokens, do_sample, seeded,
                         temperature, top_k, seed, top_p, penalty, bans, lp_n, stopping_criteria, eos, pad, warp=None):
        """generate with guidance_scale g: one left-padded prefill of the prompts and the negative prompts (clips B ..
        2B-1), then the device loops with the guidance table set (greedy and seeded calls; stopping criteria keep
        _host_stops' chunking), or _stepwise with the combination on the host (unseeded sampling). The prompts' entries
        of the sampling, ban and log-prob tables are set as an unguided call sets them; the negative clips' entries
        stay greedy and off. Returns the prompts' rows; the cache is left as after an unguided call on the prompts
        (padded by `shift` more columns when a negative prompt is longer), which generate_continue continues."""
        B, S = ids.shape
        ids2, pads2, spans, f2, shift = self._guided_batch(ids, pads, feats, neg_ids, neg_mask, neg_feats, eng.NV)
        S2 = ids2.shape[1]
        ctx = ids2[:B]                           # the prompts as the cache holds them
        n = min(max_new_tokens, self._max_seq - S2)
        if n <= 0:
            raise ValueError(f"prompt length {S2} leaves no room in max_seq {self._max_seq}")
        self._pads = pads2[:B] if pads2 else None
        self._shift = shift
        if do_sample and not seeded:
            _, logits, _ = eng.prefill(ids2, f2, spans, want_logits=True, want_token=False, n_pad=pads2)
            self._pos = S2
            self._last_out = self._stepwise(eng, ctx, logits, n, do_sample, temperature, stopping_criteria, eos, pad,
                                            top_k, top_p, penalty, bans, guidance=g, warpers=warp)
            return self._last_out[:, shift:]
        clips = list(range(B))
        if seeded:
            samp = self._sampling(eng, clips, [temperature] * B, [top_k] * B, [seed + b for b in clips], top_p, penalty,
                                  warp)
        elif penalty != 1.0:
            samp = self._sampling(eng, clips, [0.0] * B, [0] * B, [0] * B, 1.0, penalty)
        else:
            samp = contextlib.nullcontext()
        if penalty != 1.0:
            self._token_sets(eng, [(b, ids[b]) for b in clips])
        if bans:   # the extra padding columns hold no token (-1 matches no n-gram or word)
            self._histories(eng, [(b, torch.cat([torch.full((shift,), -1, dtype=torch.int64, device=ids.device), ids[b]]))
                                  for b in clips])
        with samp, self._banning(eng, clips, bans, eos, S2 + (bans.min_new if bans else 0)), \
                self._logprobs(eng, clips, lp_n), self._guiding(eng, B, g):
            if eos is None and not stopping_criteria:
                new = eng.generate(ids2, f2, spans, n, n_pad=pads2)[:B]
                self._pos = S2 + n - 1
                self._last_out = torch.cat([ctx, new.to(torch.int64)], dim=1)
            else:
                first = eng.generate(ids2, f2, spans, min(n, self._GREEDY_CHUNK), n_pad=pads2)[:B]
                self._last_out = self._host_stops(eng, ctx, first, n, stopping_criteria, eos, pad, guided=True)
        if lp_n is not None:   # the token after the prompt takes position S2 - n_pad[b]
            self.last_logprobs = self._read_logprobs(eng, self._last_out[:, S2:].cpu(),
                                                     [S2 - (pads2[b] if pads2 else 0) for b in range(B)], lp_n, eos)
        return self._last_out[:, shift:]

    # beam-search steps per vcl_llm_beam_decode call between two host-side replays (see _beam_generate). Measured with
    # tools/bench_beams.py (7B shapes, one clip at S = 448, 4 beams, 256 tokens, H100 at 700 W): 6.38 / 6.11 / 6.06 /
    # 5.96 ms per token at 4 / 8 / 16 / 32 (an earlier run: 6.24 / 5.89 / 5.91 / 5.83) -- 8 and longer are within
    # run-to-run spread, and 16 wastes at most 15 steps after an early stop
    _BEAM_CHUNK = 16

    def _beam_args(self, num_beams, num_return_sequences, length_penalty, early_stopping, do_sample, seed, logprobs,
                   top_p, repetition_penalty, stopping_criteria, bans=(None, None, None)):
        """Checks the beam-search arguments of generate on the host -> None (no beams), or (num_beams,
        num_return_sequences, length_penalty, early_stopping)"""
        if isinstance(num_beams, bool) or not isinstance(num_beams, int) or num_beams < 1:
            raise ValueError(f"generate: num_beams {num_beams!r} must be an int >= 1")
        if num_beams == 1:
            return None                         # (num_return_sequences keeps its old treatment: ignored)
        v = num_return_sequences
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise ValueError(f"generate: num_return_sequences {v!r} must be an int >= 1")
        if num_beams > vn.BEAM_MAX:
            raise ValueError(f"generate: num_beams {num_beams} exceeds {vn.BEAM_MAX}, the most the device keeps per prompt")
        if num_return_sequences > num_beams:
            raise ValueError(f"generate: num_return_sequences ({num_return_sequences}) has to be smaller or equal to "
                             f"num_beams ({num_beams})")
        if not (early_stopping is True or early_stopping is False or early_stopping == "never"):
            raise ValueError(f"generate: early_stopping {early_stopping!r} must be True, False or \"never\"")
        lp = float(length_penalty)
        if not math.isfinite(lp):
            raise ValueError(f"generate: length_penalty {length_penalty} must be finite")
        for name, bad in (("do_sample=True", do_sample), ("seed", seed is not None), ("logprobs", logprobs is not None),
                          ("top_p", float(top_p) < 1.0), ("repetition_penalty", float(repetition_penalty) != 1.0),
                          ("stopping_criteria", bool(stopping_criteria)), ("no_repeat_ngram_size", bool(bans[0])),
                          ("bad_words_ids", bans[1] is not None), ("min_new_tokens", bool(bans[2]))):
            if bad:
                raise NotImplementedError(f"generate: {name} is not supported with num_beams > 1 (beam search runs "
                                          "greedy, do_sample=False, without logits processors or stopping criteria)")
        if self.config.vocab_size > vn.SAMPLE_WIDE_MAX_V:
            raise ValueError(f"generate: beam search takes a vocabulary of at most {vn.SAMPLE_WIDE_MAX_V} tokens on the "
                             f"device, this model has {self.config.vocab_size}")
        return num_beams, num_return_sequences, lp, early_stopping

    def _beam_generate(self, input_ids, feats, attention_mask, max_new_tokens, eos_token_id, pad_token_id, k, m,
                       length_penalty, early_stopping):
        """generate(num_beams=k): HF's _beam_search (do_sample=False). The device prefills each prompt once, runs the
        per-step selection (steps 1-3 of DESIGN.md section 3, "Beam search") and forks the KV cache, in chunks of
        _BEAM_CHUNK steps from one CUDA graph; after each chunk _BeamReplay replays steps 4-6 (finished hypotheses,
        length penalty, early stopping) in fp32 torch on the records it read back, and the call stops where HF stops.
        The running beams come from the device's picks, so host and cache cannot disagree. Steps the device ran past
        HF's stop are discarded."""
        pads = left_padding(attention_mask, input_ids.shape)
        self.last_logprobs = self.last_beam_scores = None
        B, S = input_ids.shape
        if B * k > self._max_batch:
            raise ValueError(f"generate: {B} prompts x num_beams {k} = {B * k} beams exceed max_batch {self._max_batch} "
                             "(every beam takes a cache clip)")
        n = int(max_new_tokens)
        if n < 1 or S + n > self._max_seq:
            # (greedy calls cut max_new_tokens to fit; a beam call cannot: max_length decides when every candidate
            # finishes and normalizes the length penalty, so a shorter call is a different search)
            raise ValueError(f"generate: prompt length {S} + max_new_tokens {max_new_tokens} must fit max_seq "
                             f"{self._max_seq} with beams")
        eng = self._ensure_engine(need_llm=True)
        dev = self.device
        ids = input_ids.to(dev).to(torch.int64)
        vs = self._spans_dev(ids, feats, eng.NV, pads, device=dev)
        if feats is not None:
            feats = feats.to(dev)
        eos, pad = self._eos_pad(eos_token_id, pad_token_id)
        replay = _BeamReplay(B, k, S, n, eos, pad, length_penalty, early_stopping)
        self._last_out, self._after_beams = None, True
        rec, picks = eng.beam_start(ids, feats, vs, k, n, -1 if eos is None else eos, n_pad=pads)
        while not replay.steps(rec, picks):
            rec, picks = eng.beam_decode(min(self._BEAM_CHUNK, n - replay.t))
        seqs, scores = replay.result(m)
        self.last_beam_scores = scores
        return torch.cat([ids.repeat_interleave(m, dim=0), seqs.to(dev)], dim=1)

    def _contrastive_args(self, penalty_alpha, top_k, do_sample, seed, num_beams, guidance_scale, logprobs, top_p,
                          repetition_penalty, bans):
        """Checks the contrastive-search arguments of generate on the host -> None (off), or (penalty_alpha,
        top_k). Off as in HF: penalty_alpha None or 0, or top_k <= 1."""
        if penalty_alpha is None:
            return None
        if isinstance(penalty_alpha, bool) or not isinstance(penalty_alpha, (int, float)) or \
                not 0.0 <= float(penalty_alpha) <= 1.0:
            raise ValueError(f"generate: penalty_alpha {penalty_alpha!r} must be a number in [0, 1]")
        if isinstance(top_k, bool) or not isinstance(top_k, int):
            raise ValueError(f"generate: top_k {top_k!r} must be an int")
        if float(penalty_alpha) == 0.0 or top_k <= 1:
            return None
        for name, bad in (("do_sample=True", do_sample), ("seed", seed is not None),
                          ("num_beams > 1", not (isinstance(num_beams, int) and num_beams == 1)),
                          ("guidance_scale", guidance_scale is not None and float(guidance_scale) != 1.0),
                          ("logprobs", logprobs is not None), ("top_p", float(top_p) < 1.0),
                          ("repetition_penalty", float(repetition_penalty) != 1.0),
                          ("no_repeat_ngram_size", bool(bans[0])), ("bad_words_ids", bans[1] is not None),
                          ("min_new_tokens", bool(bans[2]))):
            if bad:
                raise NotImplementedError(f"generate: {name} is not supported with penalty_alpha (contrastive search "
                                          "ranks greedy candidates, do_sample=False, without other logits processors)")
        if top_k > vn.CS_MAX_K:
            raise ValueError(f"generate: top_k {top_k} exceeds {vn.CS_MAX_K}, the most contrastive-search candidates "
                             "the device ranks per prompt")
        if self.config.vocab_size > vn.SAMPLE_WIDE_MAX_V:
            raise ValueError(f"generate: contrastive search takes a vocabulary of at most {vn.SAMPLE_WIDE_MAX_V} tokens "
                             f"on the device, this model has {self.config.vocab_size}")
        return float(penalty_alpha), top_k

    def _contrastive_generate(self, input_ids, feats, attention_mask, max_new_tokens, stopping_criteria, eos_token_id,
                              pad_token_id, alpha, k):
        """generate(penalty_alpha=alpha, top_k=k): HF 4.x's _contrastive_search. The device prefills each prompt once,
        keeping its final-norm rows as the context, then every step decodes the k candidates of each prompt in k
        cache clips, ranks them, appends the winner's row to the context and copies its cache column into the other
        clips (vcl_llm_contrastive_start / _decode; one CUDA graph per chunk). EOS, padding and stopping criteria
        are applied on the host between chunks of _GREEDY_CHUNK tokens, token by token, as for seeded sampling.
        Returns [B, S + m] like greedy generate."""
        pads = left_padding(attention_mask, input_ids.shape)
        B, S = input_ids.shape
        if B * k > self._max_batch:
            raise ValueError(f"generate: {B} prompts x top_k {k} = {B * k} candidates exceed max_batch "
                             f"{self._max_batch} (contrastive search decodes every candidate in a cache clip of its "
                             "own: pass a smaller top_k or build the model with a larger max_batch)")
        n = min(int(max_new_tokens), self._max_seq - S)   # (every step decodes its candidates at column S + t)
        if n <= 0:
            raise ValueError(f"prompt length {S} leaves no room in max_seq {self._max_seq}")
        self.last_logprobs = self.last_beam_scores = None
        self._after_beams = False
        eng = self._ensure_engine(need_llm=True)
        dev = self.device
        ids = input_ids.to(dev).to(torch.int64)
        vs = self._spans_dev(ids, feats, eng.NV, pads, device=dev)
        if feats is not None:
            feats = feats.to(dev)
        eos, pad = self._eos_pad(eos_token_id, pad_token_id)
        self._last_out, self._after_contrastive = None, True
        tok, _ = eng.contrastive_start(ids, feats, vs, k, alpha, n, n_pad=pads)
        c = n if eos is None and not stopping_criteria else min(n, self._GREEDY_CHUNK)
        if c > 1:
            tok = torch.cat([tok, eng.contrastive_decode(c - 1)[0]])
        if eos is None and not stopping_criteria:
            return torch.cat([ids, tok.T.to(torch.int64)], dim=1)
        return self._host_stops(eng, ids, tok.T, n, stopping_criteria, eos, pad,
                                more=lambda m: eng.contrastive_decode(m)[0].T)

    def _host_stops(self, eng, out, new, n, stopping_criteria, eos, pad, guided=False, more=None):
        """The device-sampled loop of generate / generate_continue: `new` [B, c] int32 holds the first c tokens
        after the context `out` [B, L] (the first at column L). _stepwise's EOS / padding / stopping-criteria
        logic runs token by token over each chunk on the host; the device decodes the next _GREEDY_CHUNK tokens
        from the last kept (padded) token until a rule stops or n tokens are out. Returns [B, L + k]; self._pos
        ends at L + k - 1, where _stepwise leaves it (columns decoded past the stop are overwritten by a
        continuation). The sequence lives in one [B, L + n] buffer on out's device, filled by one copy per chunk;
        a stopping criterion is called with a view of its first L + j columns, so a call costs no copy.
        guided: clips B .. 2B-1 decode the negative prompts next to the B rows and are fed the same tokens.
        more(m): the next m tokens [B, m] of a device loop that keeps its own state (contrastive search), instead of
        decode_loop from the last kept token."""
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
            if more is not None:
                new = more(m)
                continue
            last = full[:, L + k - 1].to(torch.int32).contiguous()
            if guided:
                last = torch.cat([last, last])
            new = eng.decode_loop(last, L + k - 1, m + 1)[:B, 1:]
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
                          chunked_prefill=False, logprobs=None, top_p=1.0, repetition_penalty=1.0, no_repeat_ngram_size=None,
                          bad_words_ids=None, min_new_tokens=None, min_p=None, typical_p=None, epsilon_cutoff=None,
                          eta_cutoff=None):
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
        flight follow their actual lengths: see inflight.PagedSlots. The results are the same bit for bit; afterwards
        self.last_kv_stats holds the preemptions, the bytes swapped out and the peak blocks in use.
        chunked_prefill: on a paged model, prompts longer than _PACKED_MAX_S tokens (up to max_seq - max_new_tokens)
        are prefilled in chunks of _PACKED_MAX_S rows (inflight.prefill_chunked), not rejected; last_kv_stats
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
        preempted (inflight.PagedSlots). Rejected before any device work: an unknown key to continue, a session key
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
        without either setting write the sampling table with set_sampling and launch what they launched before.
        no_repeat_ngram_size / bad_words_ids / min_new_tokens, or a request's own keys of those names: as in generate,
        on the device, over the request's own input_ids (a continuation: the whole conversation, whose length is where
        min_new_tokens starts counting). The slot's token history is written where its token set is; a call in which
        no request bans writes no ban table and launches what it launched before.
        min_p / typical_p / epsilon_cutoff / eta_cutoff, or a request's own keys of those names: as in generate, on the
        device, for sampled requests; they are written with the request's sampling entry at every admission, resume
        and continuation."""
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
            self._warper_args(r.get("min_p", min_p), r.get("typical_p", typical_p),
                              r.get("epsilon_cutoff", epsilon_cutoff), r.get("eta_cutoff", eta_cutoff), f"request {i}",
                              r.get("do_sample", do_sample))
        eos, _ = self._eos_pad(eos_token_id, None)
        for i, r in enumerate(requests):
            r = r if isinstance(r, dict) else {}
            self._ban_args(r.get("no_repeat_ngram_size", no_repeat_ngram_size), r.get("bad_words_ids", bad_words_ids),
                           r.get("min_new_tokens", min_new_tokens), eos, f"request {i}")
        cap = self._n_slots
        n_slots = cap if slots is None else int(slots)
        if not 1 <= n_slots <= cap:
            if self._max_slots:
                raise ValueError(f"slots={slots} outside 1..{cap} (max_slots {self._max_slots})")
            raise ValueError(f"slots={slots} outside 1..{cap} (at most 16 and at most max_batch {self._max_batch})")
        eng = self._ensure_engine(need_llm=True)
        samp = dict(do_sample=do_sample, temperature=temperature, top_k=top_k, seed=seed, logprobs=logprobs, top_p=top_p,
                    repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size,
                    bad_words_ids=bad_words_ids, min_new_tokens=min_new_tokens, eos=eos, min_p=min_p,
                    typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff)
        reqs = [inflight.request(self, i, r, max_new_tokens, stopping_criteria, eng.NV, samp)
                for i, r in enumerate(requests)]
        if self._kv_blocks:
            inflight.bind_sessions(self, reqs)
            inflight.check_paged(self, reqs, chunked_prefill)
        sampling = any(r.temperature > 0 or r.penalty != 1.0 or r.bans is not None for r in reqs)
        banning = any(r.bans is not None for r in reqs)
        self._last_out, self._pos, self.last_logprobs = None, 0, None
        n_slots = min(n_slots, len(reqs))
        lps = inflight.RequestLogprobs(self, eng, reqs, n_slots)
        try:
            out = inflight.schedule(self, eng, reqs, n_slots, packed_admission, sampling, eos,
                                    chunked_prefill and bool(self._kv_blocks), lps)
            if lps.on:
                self.last_logprobs = lps.result()
            return out
        finally:
            if sampling:
                eng.set_sampling(list(range(n_slots)), [0.0] * n_slots, [0] * n_slots, [0] * n_slots)
            if banning:
                self._set_bans(eng, list(range(n_slots)), [None] * n_slots, eos, [0] * n_slots)
            if lps.on:
                eng.set_logprobs(list(range(n_slots)), [-1] * n_slots)

    @torch.no_grad()
    def score_candidates(self, input_ids, candidates, video_spatio_temporal_features=None, attention_mask=None):
        """Rank candidate answers by log-likelihood with one prefill per prompt (multiple-choice video QA).

        input_ids: B prompts, a [B, S] tensor (left-padded with attention_mask, as generate takes them; the padding is
        stripped on the host) or a list of B 1-D prompts. candidates[b]: the n_b >= 1 options of prompt b, each a 1-D
        sequence of at least one token id (text only). video_spatio_temporal_features: None, [B, NV, C], or a list of B
        entries (each [NV, C] or None).
        Returns, per prompt, dict(logprob=float64 [n_b], greedy=bool [n_b], token_logprobs=[float32 [L_bj], ...]):
        lm-eval's loglikelihood (the summed log-prob and whether every token is greedy) plus the per-token values. The
        log-prob of option token c_t is the greedy log-prob rule of generate(logprobs=...) on the bf16 logits row that
        predicts it, (x - m) - logf(W) in fp32; greedy means every c_t is the lowest-index arg-max of its row; a row
        without a finite maximum gives NaN and greedy False; logprob sums the per-token values in float64, in order.
        Each prompt is prefilled once into a cache slot, its columns are copied into the slots of its other options,
        and the options of up to max_slots sequences run as one packed continuation (candidates.py). An option's values
        do not depend on its slot, its neighbours, the prompt order or how the call is split into rounds.
        Rejected before any device work, naming the prompt and option: an empty option list or option, an id outside
        the vocabulary, a video placeholder id inside an option, an option over 512 tokens, a prompt plus option longer
        than max_seq, and features whose shapes do not match the prompts. Afterwards there is no turn for
        generate_continue to continue. A paged model raises NotImplementedError."""
        self._not_paged("score_candidates")
        eng = self._ensure_engine(need_llm=True)
        q = candidate_scoring.check(self, input_ids, candidates, video_spatio_temporal_features, attention_mask,
                                    eng.NV)
        self._last_out, self._pos, self.last_logprobs = None, 0, None
        self._after_beams, self._after_contrastive, self.last_beam_scores = False, False, None
        return candidate_scoring.score(self, eng, q)

    def end_session(self, key=None):
        """Forget the conversation kept under `key` (every kept conversation when None): its cache blocks return to
        the free list of the next generate_requests call, and a copy swapped to host memory is dropped."""
        if key is None:
            self._sessions.clear()
            return
        if key not in self._sessions:
            raise ValueError(f"end_session: no conversation is kept under key {key!r}")
        del self._sessions[key]

    def generate_continue(self, new_input_ids, do_sample=False, temperature=1.0, max_new_tokens=32,
                          stopping_criteria=None, eos_token_id="config", pad_token_id=None, top_k=50, seed=None,
                          logprobs=None, top_p=1.0, repetition_penalty=1.0, no_repeat_ngram_size=None, bad_words_ids=None,
                          min_new_tokens=None, min_p=None, typical_p=None, epsilon_cutoff=None, eta_cutoff=None):
        """Next turn about the SAME video(s): `new_input_ids` [B, S_new] follow everything generated
        so far. Only the tokens the KV cache does not hold yet (the last generated token and the new
        text) are prefilled (vcl_llm_prefill_append); the reference re-runs the tower and the whole
        prompt every turn (chat.py:137-154). Returns the full sequence [B, S_total + n] like generate.
        After a left-padded generate the cache stays padded, so every row continues its own positions; the
        new text of every row has the same length S_new (no padding inside a turn).
        seed: do_sample=True samples on the device as generate(seed=...) does. logprobs: as in generate, for the new
        tokens of this turn. top_p / repetition_penalty: as in generate; the penalty's tokens are the whole
        conversation (every earlier turn, its answers as returned, and the new text). no_repeat_ngram_size /
        bad_words_ids / min_new_tokens: as in generate, over the whole conversation; min_new_tokens counts this turn's
        tokens (HF's prompt length is the conversation's). min_p / typical_p / epsilon_cutoff / eta_cutoff: as in
        generate."""
        self._not_paged("generate_continue")
        self.last_beam_scores = None
        if getattr(self, "_after_beams", False):
            raise ValueError("generate_continue: the last generate() ran beam search (num_beams > 1), which returns "
                             "several hypotheses per prompt and leaves no single turn to continue")
        if getattr(self, "_after_contrastive", False):
            raise ValueError("generate_continue: the last generate() ran contrastive search (penalty_alpha), which "
                             "generate_continue does not continue; start the next turn with generate()")
        if getattr(self, "_last_out", None) is None:
            raise ValueError("generate_continue: no previous generate() to continue")
        lp_n = self._logprobs_arg(logprobs, "generate_continue")
        if lp_n is not None and do_sample and seed is None:
            raise NotImplementedError("generate_continue: logprobs are computed by the device sampler, and sampling "
                                      "there needs seed= (unseeded do_sample=True draws from torch's RNG on the host)")
        self.last_logprobs = None
        top_p, penalty = self._nucleus_args(top_p, repetition_penalty, "generate_continue", do_sample,
                                            device=not do_sample or seed is not None)
        warp = self._warper_args(min_p, typical_p, epsilon_cutoff, eta_cutoff, "generate_continue",
                                 do_sample and float(temperature) > 0, device=seed is not None)
        eos, pad = self._eos_pad(eos_token_id, pad_token_id)
        bans = self._ban_args(no_repeat_ngram_size, bad_words_ids, min_new_tokens, eos, "generate_continue",
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
        if seeded or lp_n is not None or ((penalty != 1.0 or bans) and not do_sample):
            B, L = ctx.shape
            clips = list(range(B))
            if seeded:
                samp = self._sampling(eng, clips, [temperature] * B, [top_k] * B, [seed + b for b in clips], top_p,
                                      penalty, warp)
            elif penalty != 1.0:   # greedy entries with the penalty
                samp = self._sampling(eng, clips, [0.0] * B, [0] * B, [0] * B, 1.0, penalty)
            else:
                samp = contextlib.nullcontext()
            if penalty != 1.0:
                self._token_sets(eng, [(b, ctx[b]) for b in clips])
            if bans:
                self._histories(eng, [(b, ctx[b]) for b in clips])
            with samp, self._banning(eng, clips, bans, eos, L + (bans.min_new if bans else 0)), \
                    self._logprobs(eng, clips, lp_n):
                _, _, tok = eng.prefill_append(tail, start)
                first = eng.decode_loop(tok, ctx.shape[1], min(n, self._GREEDY_CHUNK))
                self._last_out = self._host_stops(eng, ctx, first, n, stopping_criteria, eos, pad)
            if lp_n is not None:   # the cache keeps the padding of the generate it continues
                pads = self._pads
                self.last_logprobs = self._read_logprobs(eng, self._last_out[:, L:].cpu(),
                                                         [L - (pads[b] if pads else 0) for b in range(B)], lp_n, eos)
            return self._continued()
        _, logits, _ = eng.prefill_append(tail, start, want_logits=True, want_token=False)
        self._pos = ctx.shape[1]
        self._last_out = self._stepwise(eng, ctx, logits, n, do_sample, temperature, stopping_criteria, eos, pad, top_k,
                                        top_p, penalty, bans, warpers=warp)
        return self._continued()

    def _continued(self):
        """generate_continue's result: the conversation without the padding columns a guided generate added"""
        shift = getattr(self, "_shift", 0)
        return self._last_out[:, shift:] if shift else self._last_out

    @staticmethod
    def _host_processors(out, logits, sampled, temperature, top_k, top_p, penalty, bans=None, S=0, warpers=None):
        """HF's logits processors of the stepwise path, in HF's order, on logits [B, V] fp32 after the ids `out`
        [B, L]: RepetitionPenaltyLogitsProcessor, the banned tokens (_host_bans, with `bans` from _ban_args; the call's
        first new token at column S), then (sampled only) TemperatureLogitsWarper, TopKLogitsWarper,
        TopPLogitsWarper and the warpers of `warpers` (_host_warpers) (min_tokens_to_keep 1); a dropped token is
        -inf"""
        if penalty != 1.0:
            ids = out.to(logits.device)
            sc = torch.gather(logits, 1, ids)
            sc = torch.where(sc < 0, sc * penalty, sc / penalty)
            logits = logits.scatter(1, ids, sc)
        if bans is not None:
            logits = VideoChatGPTLlamaForCausalLM._host_bans(out, logits, bans, S)
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
        if warpers is not None:
            lg = VideoChatGPTLlamaForCausalLM._host_warpers(lg, warpers)
        return lg

    @staticmethod
    def _host_warpers(lg, warpers):
        """HF's MinPLogitsWarper, TypicalLogitsWarper, EpsilonLogitsWarper and EtaLogitsWarper (min_tokens_to_keep 1)
        on scores lg [B, V] fp32, in HF's order and with HF's torch operations; warpers: _warper_args' tuple (off: min_p
        0, typical_p 1, epsilon 0, eta 0)"""
        mp, ty, ep, et = warpers
        ninf = float("-inf")
        if mp > 0.0:
            probs = torch.softmax(lg, dim=-1)
            drop = probs < mp * probs.amax(dim=-1, keepdim=True)
            drop.scatter_(-1, torch.topk(probs, 1, dim=-1).indices, False)
            lg = lg.masked_fill(drop, ninf)
        if ty < 1.0:
            normalized = torch.nn.functional.log_softmax(lg, dim=-1)
            ent = -(normalized * torch.exp(normalized)).nansum(-1, keepdim=True)
            srt, idx = torch.sort(torch.abs((-normalized) - ent), descending=False)
            last = (lg.gather(-1, idx).softmax(dim=-1).cumsum(dim=-1) < ty).sum(dim=1)
            last.clamp_(max=srt.shape[-1] - 1)
            drop = srt > srt.gather(1, last.view(-1, 1))
            drop[..., :1] = False
            lg = lg.masked_fill(drop.scatter(1, idx, drop), ninf)
        if ep > 0.0:
            drop = (lg.softmax(dim=-1) < ep) & (lg < torch.topk(lg, 1)[0][..., -1, None])
            lg = lg.masked_fill(drop, ninf)
        if et > 0.0:
            e = torch.tensor(et, device=lg.device)
            entropy = torch.distributions.Categorical(logits=lg).entropy()
            eta = torch.min(e, torch.sqrt(e) * torch.exp(-entropy))[..., None]
            drop = (lg.softmax(dim=-1) < eta) & (lg < torch.topk(lg, 1)[0][..., -1, None])
            lg = lg.masked_fill(drop, ninf)
        return lg

    def _stepwise(self, eng, out, logits, n, do_sample, temperature, stopping_criteria, eos, pad, top_k=50, top_p=1.0,
                  penalty=1.0, bans=None, guidance=None, warpers=None):
        """One token per C-ABI call. After the loop the cache holds every returned token but the last
        (self._pos = out.shape[1] - 1), the state generate_continue starts from. The logits go through HF's
        processors in HF's order: repetition penalty (over `out` so far), the banned tokens, then temperature, top-k
        and top-p. guidance: the scale of a guided call, whose logits hold the B rows and then their B negative
        prompts (clips B .. 2B-1); HF's guidance runs first, and the negative clips are fed the same tokens."""
        S = out.shape[1]
        B = out.shape[0]
        unfinished = torch.ones(out.shape[0], dtype=torch.bool, device=out.device)
        for step in range(n):
            if guidance is not None:
                logits = self._host_guidance(logits[:B], logits[B:], guidance)
            lg = self._host_processors(out, logits, do_sample and temperature > 0, temperature, top_k, top_p, penalty,
                                       bans, S, warpers)
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
            feed = nxt.to(torch.int32)
            if guidance is not None:
                feed = torch.cat([feed, feed])
            logits, _ = eng.decode_step(feed.contiguous(), self._pos, want_logits=True)
            self._pos += 1
        return out

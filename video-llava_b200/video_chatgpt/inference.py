"""Single-clip inference (reference: video_chatgpt/inference.py).

    get_spatio_temporal_features_torch(features)            :13-44
    video_chatgpt_infer(video_frames, question, ...)         :47-125

Same signatures and return values. The pooling runs in libvcl (vcl_st_pool); the tower call and
generate go through the shim classes of video_chatgpt.model.
"""
import torch

import vcl_native as vn

from .constants import (DEFAULT_TRANSCRIPT_START, DEFAULT_VID_END_TOKEN, DEFAULT_VID_START_TOKEN,
                        DEFAULT_VIDEO_PATCH_TOKEN)
from .model.utils import KeywordsStoppingCriteria
from .video_conversation import SeparatorStyle, conv_templates


def get_spatio_temporal_features_torch(features: torch.Tensor) -> torch.Tensor:
    """[T,P,C] fp16|bf16 CUDA tensor -> [100+P, C] fp16 on the same device: per-frame means over the
    patches (zero rows up to 100), then per-patch means over the frames. T > 100 is rejected (the
    reference would silently return T+P rows, which no caller can consume)."""
    if not features.is_cuda:
        raise vn.VclError("get_spatio_temporal_features_torch: features must live on the GPU (no CPU fallback)")
    if features.dtype not in (torch.float16, torch.bfloat16):
        features = features.half()
    if features.stride(2) != 1:
        features = features.contiguous()
    return vn.st_pool(features, 100, torch.float16)


class VideoFeatureCache:
    """Pooled `[100+P, 1024]` features of the most recently used videos, by caller-chosen key.

    The reference runs the image processor and the vision tower again on every conversation turn
    about the same video (chat.py:137-147, SURVEY.md section 8f rank 4); with a key the second and later turns
    skip preprocessing, the 15.5 TFLOP tower pass and the pooling. Least recently used entries go
    first; `capacity` entries of 0.73 MB each stay on the GPU."""

    def __init__(self, capacity: int = 8):
        if capacity < 1:
            raise ValueError("VideoFeatureCache: capacity must be >= 1")
        self.capacity = capacity
        self._items = {}          # insertion-ordered: oldest first
        self.hits = 0
        self.misses = 0

    def get(self, key):
        if key in self._items:
            feats = self._items.pop(key)
            self._items[key] = feats
            self.hits += 1
            return feats
        self.misses += 1
        return None

    def put(self, key, feats):
        self._items.pop(key, None)
        self._items[key] = feats
        while len(self._items) > self.capacity:
            self._items.pop(next(iter(self._items)))

    def __len__(self):
        return len(self._items)


def video_chatgpt_infer(video_frames, question, conv_mode, model, vision_tower, tokenizer, image_processor,
                        video_token_len, transcript=None, do_sample=True, temperature=0.2, max_new_tokens=1024,
                        video_key=None, feature_cache: "VideoFeatureCache | None" = None, seed=None, top_p=1.0,
                        repetition_penalty=1.0):
    """Same flow as the reference: prompt -> tokenizer -> image processor -> tower -> pool -> generate
    -> decode. `do_sample/temperature/max_new_tokens` default to the reference's hard-coded values.
    Extension (off by default): with `video_key` and a `VideoFeatureCache`, the pooled features of a
    video are computed once and reused on later turns.
    seed (off by default): with do_sample, the tokens are sampled on the device (generate(seed=...)), reproducible
    from the seed; without one, generate samples step by step from torch's RNG as before.
    top_p / repetition_penalty (off by default, 1.0): HF's nucleus sampling and repetition penalty, passed to
    generate."""
    if model.get_model().vision_config.use_vid_start_end:
        qs = question + "\n" + DEFAULT_VID_START_TOKEN + DEFAULT_VIDEO_PATCH_TOKEN * video_token_len + DEFAULT_VID_END_TOKEN
    else:
        qs = question + "\n" + DEFAULT_VIDEO_PATCH_TOKEN * video_token_len
    if transcript:
        qs = f'{qs}\n{DEFAULT_TRANSCRIPT_START}\n"{transcript}"'
    conv = conv_templates[conv_mode].copy()
    conv.append_message(conv.roles[0], qs)
    conv.append_message(conv.roles[1], None)
    prompt = conv.get_prompt()
    inputs = tokenizer([prompt])

    feats = feature_cache.get(video_key) if (feature_cache is not None and video_key is not None) else None
    if feats is None:
        image_tensor = image_processor.preprocess(video_frames, return_tensors="pt")["pixel_values"]
        image_tensor = image_tensor.to(torch.bfloat16).cuda()
        with torch.no_grad():
            outs = vision_tower(image_tensor, output_hidden_states=True)
            frame_features = outs.hidden_states[-2][:, 1:]
        feats = get_spatio_temporal_features_torch(frame_features)
        if feature_cache is not None and video_key is not None:
            feature_cache.put(video_key, feats)

    input_ids = torch.as_tensor(inputs.input_ids).cuda()
    stop_str = conv.sep if conv.sep_style != SeparatorStyle.TWO else conv.sep2
    stopping = KeywordsStoppingCriteria([stop_str], tokenizer, input_ids)
    # HF generate stops at the tokenizer's EOS implicitly (generation config); the stop string alone
    # cannot: "</s>" tokenizes to [bos, eos] and is dropped by skip_special_tokens
    eos = getattr(tokenizer, "eos_token_id", None)
    with torch.inference_mode():
        output_ids = model.generate(input_ids, video_spatio_temporal_features=feats.unsqueeze(0),
                                    do_sample=do_sample, temperature=temperature, max_new_tokens=max_new_tokens,
                                    stopping_criteria=[stopping], eos_token_id=eos if eos is not None else "config",
                                    pad_token_id=getattr(tokenizer, "pad_token_id", None), seed=seed, top_p=top_p,
                                    repetition_penalty=repetition_penalty)
    n_diff = (input_ids != output_ids[:, :input_ids.shape[1]]).sum().item()
    if n_diff > 0:
        print(f"[Warning] {n_diff} output_ids are not the same as the input_ids")
    outputs = tokenizer.batch_decode(output_ids[:, input_ids.shape[1]:], skip_special_tokens=True)[0]
    return outputs.strip().rstrip(stop_str).strip()

"""Model / tower / tokenizer construction and frame sampling
(reference: video_chatgpt/eval/model_utils.py).

    load_video(vis_path, n_clips=1, num_frm=100, shape=(224,224))   :12-52  (+ device=: resize on the GPU)
    get_seq_frames(total_num_frames, desired_num_frames)            :55-79
    initialize_model(model_name, projection_path=None)              :82-150

initialize_model returns the same 5-tuple; `model` and `vision_tower` are the libvcl-backed shims
(one shared handle). Checkpoints must be local directories (there is no hub access on this path):
model_name/config.json + weights (+ tokenizer files), and config.mm_vision_tower a local CLIP
directory with config.json + weights (+ preprocessor_config.json).
"""
import os

import numpy as np
import torch

import vcl_native as vn

from ..constants import DEFAULT_VID_END_TOKEN, DEFAULT_VID_START_TOKEN, DEFAULT_VIDEO_PATCH_TOKEN
from ..model import VideoChatGPTLlamaForCausalLM


def get_seq_frames(total_num_frames, desired_num_frames):
    """Midpoints of `desired_num_frames` equal segments of [0, total-1] (round-half-even like np.round)."""
    seg = float(total_num_frames - 1) / desired_num_frames
    edges = [int(np.round(seg * i)) for i in range(desired_num_frames + 1)]
    return [(edges[i] + edges[i + 1]) // 2 for i in range(desired_num_frames)]


def load_video(vis_path, n_clips=1, num_frm=100, shape=(224, 224), device=None):
    """<= num_frm uniformly sampled frames as PIL images, nearest-neighbour resized to `shape`.
    With a device (e.g. "cuda"), the sampled frames are uploaded at their native size and resized there
    (vcl_resize_frames): the result is a uint8 [T,h,w,3] tensor on the device, equal to
    np.stack(load_video(...)) of the default path."""
    try:
        from decord import VideoReader, cpu
    except ImportError as e:                                   # decord is not in this image
        raise ImportError("load_video needs `decord` to decode video files; pass pre-decoded frames "
                          "([T,H,W,3] uint8) to the tower instead") from e
    from PIL import Image
    assert n_clips == 1
    vr = VideoReader(vis_path, ctx=cpu(0))
    total = len(vr)
    n = min(total, num_frm)
    arr = vr.get_batch(get_seq_frames(total, n)).asnumpy()
    h, w = shape
    if device is not None:
        t = torch.from_numpy(np.ascontiguousarray(arr)).to(device)
        if t.shape[1] != h or t.shape[2] != w:
            t = vn.resize_frames(t, (h, w), "nearest")
        return t
    if arr.shape[-3] != h or arr.shape[-2] != w:
        t = torch.from_numpy(arr).permute(0, 3, 1, 2).float()
        t = torch.nn.functional.interpolate(t, size=(h, w))
        arr = t.permute(0, 2, 3, 1).to(torch.uint8).numpy()
    return [Image.fromarray(arr[j]) for j in range(n)]


def _load_weight_files(directory):
    sd = {}
    for f in sorted(os.listdir(directory)):
        path = os.path.join(directory, f)
        if f.endswith(".safetensors"):
            from safetensors.torch import load_file
            sd.update(load_file(path))
        elif f.endswith(".bin") and "training" not in f:
            sd.update(torch.load(path, map_location="cpu"))
    if not sd:
        raise FileNotFoundError(f"no *.safetensors / *.bin weights in {directory}")
    return sd


def initialize_model(model_name, projection_path=None, max_batch=1, max_seq=2048, llm_weight_format="bf16",
                     max_slots=None, kv_blocks=None):
    from transformers import AutoTokenizer, CLIPImageProcessor
    model_name = os.path.expanduser(model_name)
    tokenizer = AutoTokenizer.from_pretrained(model_name)
    model = VideoChatGPTLlamaForCausalLM.from_pretrained(model_name, use_cache=True, max_batch=max_batch,
                                                         max_seq=max_seq, llm_weight_format=llm_weight_format,
                                                         max_slots=max_slots, kv_blocks=kv_blocks)
    tower_dir = model.config.mm_vision_tower
    image_processor = CLIPImageProcessor.from_pretrained(tower_dir)

    mm_use_vid_start_end = True
    tokenizer.add_tokens([DEFAULT_VIDEO_PATCH_TOKEN], special_tokens=True)
    if mm_use_vid_start_end:
        tokenizer.add_tokens([DEFAULT_VID_START_TOKEN, DEFAULT_VID_END_TOKEN], special_tokens=True)
    model.resize_token_embeddings(len(tokenizer))

    if projection_path:
        print(f"Loading weights from {projection_path}")
        status = model.load_state_dict(torch.load(projection_path, map_location="cpu"), strict=False)
        if status.unexpected_keys:
            print(f"Unexpected Keys: {status.unexpected_keys}.\nThe Video-ChatGPT weights are not loaded correctly.")
        print(f"Weights loaded from {projection_path}")

    model = model.eval().cuda()
    vision_tower = model.get_vision_tower()
    vision_tower.load_state_dict(_load_weight_files(tower_dir))
    vision_tower = vision_tower.eval()

    vc = model.get_model().vision_config
    vc.vid_patch_token = tokenizer.convert_tokens_to_ids([DEFAULT_VIDEO_PATCH_TOKEN])[0]
    vc.use_vid_start_end = mm_use_vid_start_end
    if mm_use_vid_start_end:
        vc.vid_start_token, vc.vid_end_token = tokenizer.convert_tokens_to_ids(
            [DEFAULT_VID_START_TOKEN, DEFAULT_VID_END_TOKEN])
    video_token_len = (vc.frame_size // vc.patch_size) ** 2 + 100
    return model, vision_tower, tokenizer, image_processor, video_token_len

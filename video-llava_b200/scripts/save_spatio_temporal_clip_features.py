"""Offline CLIP feature extraction (reference: scripts/save_spatio_temporal_clip_features.py).

    get_spatio_temporal_features(features, num_temporal_tokens=100)   :46-57   numpy in / numpy out
    main()                                                            :74-139  one {video_id}.pkl per video

The per-video device work is ONE C-ABI call (vcl_clip_features: ViT over all sampled frames + CLS
drop + pool), instead of the reference's 32-frame chunks with a D2H copy of every chunk; the on-disk
format is unchanged (pickle of a [100+P, 1024] float16 ndarray, resume-by-skip, flush every 512). The sampled
frames are resized on the GPU (load_video(..., device="cuda")) rather than on the CPU, with identical pixels.
"""
import argparse
import os
import pickle
import sys

import numpy as np
import torch

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)
import vcl_native as vn  # noqa: E402

FLUSH_EVERY = 512      # the reference writes its pending features every 512 processed videos (:129-134)


def get_spatio_temporal_features(features, num_temporal_tokens=100):
    """[T,P,C] float16 ndarray -> [num_temporal_tokens + P, C] float16 ndarray (pooled on the GPU)."""
    f = torch.from_numpy(np.ascontiguousarray(features)).cuda()
    if f.dtype not in (torch.float16, torch.bfloat16):
        f = f.half()
    return vn.st_pool(f, num_temporal_tokens, torch.float16).cpu().numpy()


def extract_video(engine, frames_u8) -> np.ndarray:
    """frames_u8 [T,H,W,3] uint8 ndarray or CUDA tensor (T <= 100) -> pooled [100+P, 1024] float16 ndarray."""
    px = frames_u8 if isinstance(frames_u8, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(frames_u8)).cuda()
    return engine.clip_features(px, torch.float16).cpu().numpy()


def parse_args():
    p = argparse.ArgumentParser(description="CLIP spatio-temporal feature extraction (libvcl)")
    p.add_argument("--llava", required=True, choices=["1.1", "1.5"], help="LLaVA version (224 px / 336 px tower)")
    p.add_argument("--video_dir_path", required=True)
    p.add_argument("--clip_feat_path", required=True)
    p.add_argument("--clip_dir", required=True, help="local CLIP checkpoint directory (config.json + weights)")
    p.add_argument("--infer_batch", type=int, default=32, help="accepted for CLI compatibility; unused")
    return p.parse_args()


def main():
    from video_chatgpt.eval.model_utils import _load_weight_files, load_video
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    args = parse_args()
    os.makedirs(args.clip_feat_path, exist_ok=True)
    size = 224 if args.llava == "1.1" else 336
    # tower-only engine: a zero-layer language model keeps the handle small
    owner = VideoChatGPTLlamaForCausalLM(VideoChatGPTConfig(num_hidden_layers=0, hidden_size=512, intermediate_size=1024,
                                                            num_attention_heads=4, vocab_size=8),
                                         clip_config=args.clip_dir, max_seq=8)
    tower = owner.get_vision_tower()
    tower.load_state_dict(_load_weight_files(args.clip_dir))
    engine = owner._ensure_engine(need_clip=True)
    pending, counter = {}, 0

    def flush():
        for key, feats in pending.items():
            with open(f"{args.clip_feat_path}/{key}.pkl", "wb") as f:
                pickle.dump(feats, f)
        pending.clear()

    for name in sorted(os.listdir(args.video_dir_path)):
        vid = name.split(".")[0]
        if os.path.exists(f"{args.clip_feat_path}/{vid}.pkl"):
            continue
        try:
            # the native frames go to the GPU and are resized there (load_video's nearest rule, bit for bit)
            frames = load_video(f"{args.video_dir_path}/{name}", shape=(size, size), device="cuda")
            pending[vid] = extract_video(engine, frames)
            counter += 1
        except Exception as e:
            print(f"Can't process {args.video_dir_path}/{name}: {e}")
        if counter % FLUSH_EVERY == 0:
            flush()
    flush()


if __name__ == "__main__":
    main()

"""Frame preprocessing on the CPU against the device resize (vcl_resize_frames).

    python tools/bench_frames.py [--frames 100] [--sizes 224,336] [--res 480p,720p,1080p] [--reps 10] [--out DIR]

100 seeded random frames per native resolution (480p = 854x480, 720p, 1080p), towers of 224 and 336 px. Per case:
  cpu_load_video_s    load_video's resize on the CPU (float copy, nearest interpolate to size x size, back to uint8)
  cpu_processor_s     the installed image processor on those resized frames (its resize is then a no-op)
  cpu_pipeline_s      the two together: what every caller pays today before the GPU starts
  cpu_pil_native_s    PIL's bicubic shortest-edge resize + center crop of the native frames (the processor's resize
                      and crop when callers pass native frames, as transformers pinned by the reference does it)
  h2d_ms              torch.from_numpy(native).cuda() of the pageable frames, ended by a synchronise
  nearest_ms          vn.resize_frames(native, (size, size), "nearest"): load_video(device="cuda")'s resize
  bicubic_ms          processor_resize(native): the processor's resize + crop on the device
  features_ms         clip_features end to end from native host frames: H2D, bicubic resize + crop, the ViT-L/14
                      tower (23 layers, random weights) and the pool, ended by a synchronise
  features_resized_ms clip_features from frames already at the crop size on the device (the tower and pool alone)
Device numbers are the median over --reps calls after one warm-up, each a host clock around work ended by a
synchronise. Prints one JSON line per case with the card and power limit.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "video-llava_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

import vcl_native as vn  # noqa: E402
from bench_padded import card  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from video_chatgpt.preprocess import processor_plan, processor_resize  # noqa: E402

RES = {"480p": (480, 854), "720p": (720, 1280), "1080p": (1080, 1920)}


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def make_engine(size, n_frames):
    ccfg = O.ClipCfg(image=size)
    lcfg = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=1)
    c = vn.vcl_config()
    c.clip_layers, c.clip_hidden, c.clip_inter, c.clip_heads = 23, 1024, 4096, 16
    c.image_size, c.patch_size, c.clip_ln_eps = size, 14, 1e-5
    c.llm_layers, c.llm_hidden, c.llm_inter, c.llm_heads = 1, 512, 1024, 4
    c.vocab, c.rms_eps, c.rope_theta = lcfg.vocab, 1e-5, 10000.0
    c.proj_type, c.n_temporal = vn.PROJ_LINEAR, 100
    c.max_frames, c.max_batch, c.max_seq = n_frames, 1, 8
    eng = vn.Engine(c)
    bf = lambda sd: {k: v.to("cuda", torch.bfloat16) for k, v in sd.items()}
    eng.load_clip(bf(O.random_clip_state(ccfg, seed=0, n_layers=23)))
    eng.load_llm(bf(O.random_llm_state(lcfg, seed=0)))
    return eng


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--sizes", default="224,336")
    ap.add_argument("--res", default="480p,720p,1080p")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/bench_frames.jsonl")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames.py measures the device path and needs a GPU")
    from transformers import CLIPImageProcessor
    name, power = card()
    lines = []
    for size in [int(s) for s in a.sizes.split(",")]:
        ip = CLIPImageProcessor(size={"shortest_edge": size}, crop_size={"height": size, "width": size})
        eng = make_engine(size, a.frames)
        for res in a.res.split(","):
            H, W = RES[res]
            native = np.random.default_rng(H + size).integers(0, 256, (a.frames, H, W, 3), dtype=np.uint8)
            # CPU: load_video's resize, then the processor on the resized frames
            t0 = time.perf_counter()
            t = torch.nn.functional.interpolate(torch.from_numpy(native).permute(0, 3, 1, 2).float(), size=(size, size))
            resized = t.permute(0, 2, 3, 1).to(torch.uint8).numpy()
            t_lv = time.perf_counter() - t0
            pil = [Image.fromarray(f) for f in resized]
            t0 = time.perf_counter()
            ip.preprocess(pil, return_tensors="pt")
            t_ip = time.perf_counter() - t0
            (oh, ow), (top, left, ch, cw) = processor_plan(ip, H, W, size)
            t0 = time.perf_counter()
            for f in native:
                Image.fromarray(f).resize((ow, oh), Image.BICUBIC).crop((left, top, left + cw, top + ch))
            t_pil = time.perf_counter() - t0

            dev = torch.from_numpy(native).cuda()
            h2d = timed(lambda: torch.from_numpy(native).cuda(), a.reps)
            near = timed(lambda: vn.resize_frames(dev, (size, size), "nearest"), a.reps)
            bic = timed(lambda: processor_resize(dev, ip, size), a.reps)
            feats = timed(lambda: eng.clip_features(processor_resize(torch.from_numpy(native), ip, size)), a.reps)
            ready = processor_resize(dev, ip, size)
            feats_ready = timed(lambda: eng.clip_features(ready), a.reps)
            res_line = dict(card=name, power_limit=power, frames=a.frames, native=f"{W}x{H}", size=size,
                            native_mb=round(native.nbytes / 1e6, 1), cpu_load_video_s=round(t_lv, 3),
                            cpu_processor_s=round(t_ip, 3), cpu_pipeline_s=round(t_lv + t_ip, 3),
                            cpu_pil_native_s=round(t_pil, 3), h2d_ms=round(h2d, 3), nearest_ms=round(near, 3),
                            bicubic_ms=round(bic, 3), features_ms=round(feats, 3),
                            features_resized_ms=round(feats_ready, 3), cpu_threads=torch.get_num_threads())
            print(json.dumps(res_line), flush=True)
            lines.append(json.dumps(res_line))
        eng.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_frames.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

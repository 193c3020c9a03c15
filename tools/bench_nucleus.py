"""Cost of top-p and the repetition penalty in the device sampler (sampling.cu): microseconds per sampler call at
V = 32 003 and B = 1, 16, 64 for the default settings (the 16-bit sampler) and, on the 32-bit sampler, the penalty,
top-p, both, and neither (p = 1, r = 1), all with top_k 50 (HF's default), and top-p over the whole vocabulary
(top_k 0). CUDA events around `--iters` launches after a warm-up; one JSON line per configuration, with the card's
name and power limit.

    python tools/bench_nucleus.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "video-llava_b200"))
import vcl_native as vn  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:   # noqa: BLE001
        return torch.cuda.get_device_name(), "unknown"


def time_us(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1000.0 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    name, limit = card()
    V = 32003
    for B in (1, 16, 64):
        g = torch.Generator().manual_seed(B)
        x = (torch.randn(B, V, generator=g) * 3).bfloat16().float().to("cuda")
        T, k, seed, ctr = [0.7] * B, [50] * B, list(range(B)), [100] * B
        sets = torch.zeros(B, vn.token_set_words(V), dtype=torch.int32, device="cuda")
        sets[:, :300] = -1                                  # 9 600 tokens in each set
        runs = {
            "default": lambda: vn.op_sample(x, T, k, seed, ctr),
            "wide_off": lambda: vn.op_sample_ex(x, T, k, seed, ctr, [1.0] * B, [1.0] * B),
            "penalty": lambda: vn.op_sample_ex(x, T, k, seed, ctr, [1.0] * B, [1.2] * B, token_sets=sets),
            "top_p": lambda: vn.op_sample_ex(x, T, k, seed, ctr, [0.9] * B, [1.0] * B),
            "both": lambda: vn.op_sample_ex(x, T, k, seed, ctr, [0.9] * B, [1.2] * B, token_sets=sets),
            "top_p_all_tokens": lambda: vn.op_sample_ex(x, T, [0] * B, seed, ctr, [0.9] * B, [1.0] * B),
        }
        for what, fn in runs.items():
            us = time_us(fn, args.iters)
            print(json.dumps(dict(B=B, V=V, setting=what, top_k=0 if what == "top_p_all_tokens" else 50,
                                  us_per_call=round(us, 2), card=name, power_limit=limit,
                                  note="includes the host-to-device copy of the per-row settings")), flush=True)


if __name__ == "__main__":
    main()

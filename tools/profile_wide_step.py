"""Per-kernel split of one decode step at 17..64 clips (torch.profiler; H100; prints one JSON line).

    python tools/profile_wide_step.py [--clips 64] [--formats bf16,fp8_e4m3] [--steps 3] [--out DIR]

Vicuna-7B shapes with random weights (bench.py's), prompts of S = 448 with video, then eager decode steps at
positions 448, 449, ... (one engine per format). The kernels of the profiled steps are taken in launch order and
attributed per layer: the projections by matrix (q|k|v, o_proj, gate|up, down_proj, and the lm_head), the decode
attention, the window-major RMSNorms (xwin_norm) and the rest. Per entry: device µs per step and GB/s of the bytes it
has to move: the streamed weights (bf16 slots, or fp8 codes + row scales), plus the KV cache read for the attention;
for the projections also "act_l2_gb_s", the activation windows every CTA reads from L2 (grid x B x K x 2 bytes).
The card's name and power limit are printed with the numbers. A trace is written under --out when given.
"""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "video-llava_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402
import vcl_native as vn  # noqa: E402
from bench_fp8 import S, engine, prompts  # noqa: E402
from bench_padded import card  # noqa: E402


def attribute(names, layers):
    """kernel names of one step in launch order -> a label per kernel"""
    labels, layer, phase = [], -1, None
    proj_in_phase = []
    for i, n in enumerate(names):
        if "xwin_norm" in n:
            if phase in (None, "down"):
                layer += 1
                phase = "qkv" if layer < layers else "lm_head"
            else:
                phase = "gate|up"
            labels.append("xwin_norm")
        elif "decode_attn" in n:
            labels.append("attention")
            phase = "o_proj"
        elif "gemv_tcw" in n:
            labels.append(phase)
            if phase == "gate|up":
                proj_in_phase.append(i)
        else:
            labels.append("other")
        # the last projection launch before the next norm of a layer's MLP half is down_proj
        if phase == "gate|up" and (i + 1 == len(names) or "xwin_norm" in names[i + 1]) and proj_in_phase:
            labels[proj_in_phase[-1]] = "down_proj"
            proj_in_phase = []
            phase = "down"
    return labels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--formats", default="bf16,fp8_e4m3")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_wide_step.py needs an H100 (no CPU measurement)")
    name, power = card()
    m = bench.MODELS["7b"]
    D, F, L, V, B = m["hidden"], m["inter"], m["layers"], 32003, a.clips
    mats = {"qkv": (3 * D, D), "o_proj": (D, D), "gate|up": (2 * F, D), "down_proj": (D, F), "lm_head": (V, D)}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = {"card": name, "power_limit": power, "clips": B, "layers": L, "steps": a.steps, "split": {}}
    _, llm = bench.device_weights("7b", "cuda")
    for fmt in a.formats.split(","):
        eng, _ = engine("7b", fmt, max_batch=B, llm=llm)
        ids, vf, vs = prompts(B)
        tok = eng.prefill(ids, vf, vs)[2]
        for i in range(2):
            _, tok = eng.decode_step(tok, S + i)
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(a.steps):
                _, tok = eng.decode_step(tok, S + 2 + i)
            torch.cuda.synchronize()
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            prof.export_chrome_trace(os.path.join(a.out, f"wide_step_{fmt}_B{B}.json"))
        ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
                     and "memset" not in e.name.lower()), key=lambda e: e.time_range.start)
        per_step = len(ev) // a.steps
        us = collections.defaultdict(float)
        for s in range(a.steps):
            chunk = ev[s * per_step:(s + 1) * per_step]
            for lab, e in zip(attribute([e.name for e in chunk], L), chunk):
                us[lab] += e.time_range.elapsed_us() / a.steps
        out = {}
        for lab, t in sorted(us.items(), key=lambda kv: -kv[1]):
            row = {"us_per_step": round(t, 1)}
            if lab in mats:
                N, K = mats[lab]
                n = 1 if lab == "lm_head" else L
                wb = vn.tiled_elems(N, K) * (2 if fmt == "bf16" else 1) + (4 * N if fmt != "bf16" else 0)
                grid = min((N + 15) // 16, sms)
                row["weight_gb_s"] = round(n * wb / t / 1e3, 1)
                row["act_l2_gb_s"] = round(n * grid * B * K * 2 / t / 1e3, 1)
            elif lab == "attention":
                kv = 2 * L * B * (S + 2 + a.steps // 2) * D * 2
                row["kv_gb_s"] = round(kv / t / 1e3, 1)
            out[lab] = row
        out["total_us_per_step"] = round(sum(us.values()), 1)
        res["split"][fmt] = out
        print(f"[profile_wide_step] {fmt}: {out}", flush=True)
        eng.close()
        del eng
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(os.path.join(a.out, "profile_wide_step.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

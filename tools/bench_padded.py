"""Batched vs one-at-a-time generation of prompts of different lengths (left-padded batch).

    python tools/bench_padded.py [--clips 16] [--new 32] [--min-len 400] [--repeats 5] [--warmup 1] [--out DIR]

Vicuna-7B shapes with random-init bf16 weights (bench.device_weights, seed 0) and random video features; the
vision tower is not part of the measurement. The clips' prompts (bench.synthetic_prompt_ids with a shorter text
before the video) have lengths spread evenly over min-len .. 448. Two arms, alternated `--repeats` times after
`--warmup` rounds of both:
  (a) padded  one vcl_llm_generate_padded call over all clips (left-padded to 448), --new greedy tokens
  (b) alone   the same clips one vcl_llm_generate call each, unpadded
Each arm is timed with a host clock around its calls, ended by a stream synchronise. Prints one JSON line: ms per
clip of both arms (min and median over the repeats), the ratio alone / padded, the card name and power limit,
and whether the padded tokens match the one-at-a-time tokens under the margin rule of the parity tests: identical
up to the first step where the clip's own top-1/top-2 logit margin is below 3 bf16 ulps (from here on, two
correct bf16 paths may pick different tokens).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "video-llava_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402
import vcl_native as vn  # noqa: E402

S_MAX, N_VID = 448, 356


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # the measurement stands without it, but says so
        return torch.cuda.get_device_name(0), f"unknown ({type(e).__name__})"


def make_engine(B, n_new):
    m = bench.MODELS["7b"]
    c = vn.vcl_config()
    c.clip_layers, c.clip_hidden, c.clip_inter, c.clip_heads = 0, 1024, 4096, 16
    c.image_size, c.patch_size, c.clip_ln_eps = 224, 14, 1e-5
    c.llm_layers, c.llm_hidden, c.llm_inter, c.llm_heads = m["layers"], m["hidden"], m["inter"], m["heads"]
    c.vocab, c.rms_eps, c.rope_theta = 32003, 1e-5, 10000.0
    c.proj_type, c.n_temporal = vn.PROJ_LINEAR, 100
    c.max_frames, c.max_batch, c.max_seq = 1, B, S_MAX + n_new
    eng = vn.Engine(c)
    _, llm = bench.device_weights("7b", "cuda")
    eng.load_llm(llm)
    del llm
    torch.cuda.empty_cache()
    return eng


def prompts(B, min_len):
    """B rows with lengths spread evenly over min_len .. 448, left-padded with id 0"""
    lens = [S_MAX - round((S_MAX - min_len) * b / max(B - 1, 1)) for b in range(B)]
    rows = [bench.synthetic_prompt_ids(seed=1 + b, n_pre=63 - (S_MAX - n)).cuda() for b, n in enumerate(lens)]
    ids = torch.zeros(B, S_MAX, dtype=torch.int64, device="cuda")
    for b, r in enumerate(rows):
        ids[b, S_MAX - r.shape[1]:] = r[0]
    pads = [S_MAX - r.shape[1] for r in rows]
    vs = torch.full((B,), 64, dtype=torch.int32, device="cuda")      # <vid_start> column (64 - pad in the row alone)
    return ids, pads, vs, rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--new", type=int, default=32)
    ap.add_argument("--min-len", type=int, default=400)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/bench_padded.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_padded.py needs an H100 (no CPU measurement)")
    assert 385 + 15 <= a.min_len <= S_MAX
    B, n_new = a.clips, a.new
    name, power = card()
    eng = make_engine(B, n_new)
    ids, pads, vs, rows = prompts(B, a.min_len)
    vf = (torch.randn(B, N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7)) * 0.5
          ).to(torch.bfloat16)
    st = torch.cuda.Stream()      # the decode loop is captured into a CUDA graph on a non-default stream

    def padded():
        return eng.generate(ids, vf, vs, n_new, n_pad=pads)

    def alone():
        return [eng.generate(r, vf[b:b + 1], vs[b:b + 1] - pads[b], n_new) for b, r in enumerate(rows)]

    def timed(fn):
        st.synchronize()
        t0 = time.perf_counter()
        with torch.cuda.stream(st):
            out = fn()
        st.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    for _ in range(a.warmup):
        timed(padded)
        timed(alone)
    t_pad, t_alone = [], []
    for _ in range(a.repeats):
        t, tok_pad = timed(padded)
        t_pad.append(t / B)
        t, tok_alone = timed(alone)
        t_alone.append(t / B)

    # margin rule: each clip's own logits, step by step (greedy, so the same tokens as its generate call)
    match_full = match_to_tie = 0
    first_diff = []
    with torch.cuda.stream(st):
        for b, r in enumerate(rows):
            _, lg, tok = eng.prefill(r, vf[b:b + 1], vs[b:b + 1] - pads[b], want_logits=True)
            tie = n_new
            for i in range(n_new):
                top = torch.topk(lg[0], 2)
                ulp = top.values[0].abs().clamp_min(2 ** -6) * 2 ** -7
                if tie == n_new and ((top.values[0] - top.values[1]) / ulp).item() < 3:
                    tie = i
                if i + 1 < n_new:
                    lg, tok = eng.decode_step(tok, r.shape[1] + i, want_logits=True)
            same = (tok_pad[b] == tok_alone[b][0]).tolist()
            d = same.index(False) if False in same else n_new
            first_diff.append(d)
            match_full += d == n_new
            match_to_tie += d >= tie
    st.synchronize()
    res = {
        "what": f"{B} clips, prompt lengths {min(r.shape[1] for r in rows)}..{S_MAX}, {n_new} greedy tokens, "
                "Vicuna-7B shapes, random bf16 weights",
        "card": name, "power_limit": power,
        "padded_ms_per_clip": {"min": round(min(t_pad), 2), "median": round(statistics.median(t_pad), 2)},
        "alone_ms_per_clip": {"min": round(min(t_alone), 2), "median": round(statistics.median(t_alone), 2)},
        "speedup_alone_over_padded": round(statistics.median(t_alone) / statistics.median(t_pad), 2),
        "repeats": a.repeats, "warmup": a.warmup,
        "tokens_identical_clips": f"{match_full}/{B}",
        "tokens_match_margin_rule_clips": f"{match_to_tie}/{B}",
        "first_differing_step_per_clip": first_diff,
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_padded.json"), "w") as f:
            f.write(line + "\n")
    if match_to_tie != B:
        raise SystemExit("padded tokens differ from the one-at-a-time tokens before a near-tie")


if __name__ == "__main__":
    main()

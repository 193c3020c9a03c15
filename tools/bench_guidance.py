"""The cost of classifier-free guidance in generate (H100; one JSON line per clip count and arm).

    python tools/bench_guidance.py [--new 256] [--batches 1,2,4,8] [--reps 3]

Workload: Vicuna-7B shapes with random bf16 weights, B prompts with video of 400-448 tokens (seeded lengths, left-padded
with attention_mask), greedy, EOS off, --new tokens. Arms:
  none      no guidance
  text      guidance_scale 1.5 against each prompt without its video span (the negative video_chatgpt_infer builds)
  default   guidance_scale 1.5 against HF's default negative, each prompt's last token alone
A guided arm decodes 2B clips (every negative prompt takes a cache clip) and prefills 2B rows padded to the longest.
Each call is timed by the host clock around generate() and a stream synchronise. The prefill cost is a call of one new
token (prefill + first token). ms per token is (time of --new tokens - time of one) / (--new - 1). After one warm-up
call of each arm, which captures the graphs, the arms alternate call by call --reps times. Each line reports the
median with the min and max. The card's name and power limit are printed with the numbers.
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

import torch  # noqa: E402

import bench  # noqa: E402
from bench_inflight import N_VID, S_MAX, make_model  # noqa: E402
from bench_nucleus import card  # noqa: E402

N_POST = 26


def batch(B, seed):
    """B prompts of 400-448 tokens (1 + n_pre + video span + 26), left-padded, and the same prompts without the
    span: (ids, mask, neg_ids, neg_mask)"""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for b in range(B):
        n_pre = int(torch.randint(15, 64, (1,), generator=g))
        rows.append(bench.synthetic_prompt_ids(seed=seed + b, n_pre=n_pre)[0].cpu())
    negs = [torch.cat([r[:-(N_VID + 2 + N_POST)], r[-N_POST:]]) for r in rows]

    def pad(rs):
        S = max(len(r) for r in rs)
        ids = torch.zeros(len(rs), S, dtype=torch.int64)
        mask = torch.zeros(len(rs), S, dtype=torch.int64)
        for b, r in enumerate(rs):
            ids[b, S - len(r):] = r
            mask[b, S - len(r):] = 1
        return ids.cuda(), mask.cuda()

    return (*pad(rows), *pad(negs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    name, limit = card()
    Bs = [int(s) for s in args.batches.split(",")]
    model, _, _ = make_model(2 * max(Bs), S_MAX + args.new)
    st = torch.cuda.Stream()
    for B in Bs:
        ids, mask, neg, neg_mask = batch(B, 100 + B)
        gf = torch.Generator(device="cuda").manual_seed(7)
        feats = (torch.randn(B, N_VID, 1024, device="cuda", generator=gf) * 0.5).to(torch.bfloat16)
        arms = {"none": {}, "text": dict(guidance_scale=1.5, negative_prompt_ids=neg,
                                         negative_prompt_attention_mask=neg_mask),
                "default": dict(guidance_scale=1.5)}

        def call(kw, n):
            with torch.cuda.stream(st):
                st.synchronize()
                t0 = time.perf_counter()
                model.generate(ids, video_spatio_temporal_features=feats, attention_mask=mask, max_new_tokens=n,
                               eos_token_id=None, **kw)
                st.synchronize()
            return time.perf_counter() - t0

        for kw in arms.values():   # warm-up: graphs captured, kernels loaded
            call(kw, 1), call(kw, args.new)
        times = {a: ([], []) for a in arms}
        for _ in range(args.reps):
            for a, kw in arms.items():
                times[a][0].append(call(kw, 1))
                times[a][1].append(call(kw, args.new))
        for a in arms:
            one, full = times[a]
            per = [(f - o) * 1000.0 / (args.new - 1) for o, f in zip(one, full)]
            print(json.dumps(dict(
                clips=B, arm=arm_name(a), prompt_cols=ids.shape[1], new_tokens=args.new,
                ms_per_token=round(statistics.median(per), 3), ms_per_token_min=round(min(per), 3),
                ms_per_token_max=round(max(per), 3), prefill_ms=round(statistics.median(one) * 1000.0, 2),
                prefill_ms_min=round(min(one) * 1000.0, 2), prefill_ms_max=round(max(one) * 1000.0, 2),
                call_s=round(statistics.median(full), 3), card=name, power_limit=limit)), flush=True)


def arm_name(a):
    return {"none": "unguided", "text": "guided, text-only negative", "default": "guided, default negative"}[a]


if __name__ == "__main__":
    main()

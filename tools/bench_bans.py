"""The cost of banned tokens in the decode loop (H100; one JSON line per slot count and arm).

    python tools/bench_bans.py [--new 1024] [--slots 1,16] [--reps 2]

(One slot count per process where memory is tight: an engine's device memory is freed when the process ends.)

Workload: Vicuna-7B shapes with random bf16 weights, B clips of one prompt with video (S = 448: 356 video rows), greedy,
--new tokens: the longest histories the ban stage scans. EOS is id 32002 (<vid_end>), so every arm runs the same
device loops of 32 tokens with a host-side EOS check between them; min_new_tokens = --new keeps the last arm from
stopping early, and an arm that does stop is timed over the tokens it made. Arms:
  default   no setting (the arg-max kernels)
  penalty   repetition_penalty 1.2 (the 32-bit sampler without bans: today's cost of that sampler)
  ngram     no_repeat_ngram_size 3
  all       no_repeat_ngram_size 3, 8 bad words and min_new_tokens
ms per token = wall time of generate() (prefill included) / new tokens, the median of --reps calls after one warm-up
call that captures the graphs. The card's name and power limit are printed with the numbers.
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

EOS = 32002
WORDS = [[29871], [1576, 338], [450, 4086, 1158], [3869], [32000], [32001], [13, 13], [2]]   # 8 bad words


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=1024)
    ap.add_argument("--slots", default="1,16")   # 64 slots of 448 + 1024 columns do not fit next to the weights
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    name, limit = card()
    arms = {"default": {}, "penalty": dict(repetition_penalty=1.2), "ngram": dict(no_repeat_ngram_size=3),
            "all": dict(no_repeat_ngram_size=3, bad_words_ids=WORDS, min_new_tokens=args.new)}
    for B in [int(s) for s in args.slots.split(",")]:
        model, _, _ = make_model(B, S_MAX + args.new)
        ids = bench.synthetic_prompt_ids(seed=1, n_pre=63)[0][None].repeat(B, 1)
        g = torch.Generator(device="cuda").manual_seed(100)
        feats = (torch.randn(1, N_VID, 1024, device="cuda", generator=g) * 0.5).to(torch.bfloat16).repeat(B, 1, 1)
        st = torch.cuda.Stream()
        for arm, kw in arms.items():
            times, made = [], 0
            with torch.cuda.stream(st):
                for rep in range(args.reps + 1):
                    st.synchronize()
                    t0 = time.perf_counter()
                    out = model.generate(ids, video_spatio_temporal_features=feats, max_new_tokens=args.new,
                                         eos_token_id=EOS, **kw)
                    st.synchronize()
                    if rep:
                        times.append(time.perf_counter() - t0)
                    made = out.shape[1] - ids.shape[1]
            sec = statistics.median(times)
            print(json.dumps(dict(slots=B, arm=arm, prompt=ids.shape[1], new_tokens=made,
                                  ms_per_token=round(sec * 1000.0 / made, 3), seconds=round(sec, 3),
                                  card=name, power_limit=limit)), flush=True)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

"""Cost of the min-p, typical, epsilon and eta warpers (sampling.cu, warp_row); one JSON line per measurement, with
the card's name and power limit.

    python tools/bench_warpers.py [--iters 200] [--rounds 5] [--new 256] [--reps 6] [--skip-decode]

Sampler: microseconds per vcl_op_sample_warpers call at V = 32 003 and B = 1, 16, 64 (logits of spread 3, T 0.7) for
the default settings (the 16-bit sampler, vcl_op_sample), the 32-bit sampler with the warpers off, min-p 0.05,
typical 0.9, epsilon 3e-4, eta 3e-4 and all four together, each with top_k 50 and top_k 0 (the whole vocabulary).
CUDA events around --iters launches after a warm-up; each call includes the stream-ordered allocation, host-to-device
copy and free of its settings, which every arm but "default" makes alike. The arms alternate within each of --rounds
rounds (in reverse order every other round); each line gives the median, smallest and largest round.

Decode step: Vicuna-7B shapes with random bf16 weights, one prompt with video (S = 448), seeded sampling (T 0.7,
top_k 50, no EOS) of --new tokens, with and without min_p 0.05: generate() at 1 clip, and generate_requests() with 16
copies of the request in 16 in-flight slots. ms per step = wall time (prefill included) / new tokens; after one
warm-up call per arm that captures its graphs, the two arms alternate for --reps calls each, and each line gives the
median, smallest and largest call.
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

import vcl_native as vn  # noqa: E402
from bench_nucleus import card, time_us  # noqa: E402

SETTINGS = {"off": (0.0, 1.0, 0.0, 0.0), "min_p": (0.05, 1.0, 0.0, 0.0), "typical": (0.0, 0.9, 0.0, 0.0),
            "epsilon": (0.0, 1.0, 3e-4, 0.0), "eta": (0.0, 1.0, 0.0, 3e-4), "all": (0.05, 0.9, 3e-4, 3e-4)}


def spread(xs):
    """median, min and max of a list of timings, rounded"""
    return dict(median=round(statistics.median(xs), 2), min=round(min(xs), 2), max=round(max(xs), 2))


def sampler(iters, rounds, name, limit):
    V = 32003
    for B in (1, 16, 64):
        g = torch.Generator().manual_seed(B)
        x = (torch.randn(B, V, generator=g) * 3).bfloat16().float().to("cuda")
        T, seed, ctr = [0.7] * B, list(range(B)), [100] * B
        for k in (50, 0):
            ks = [k] * B
            arms = {"default": lambda: vn.op_sample(x, T, ks, seed, ctr)}
            for what, w in SETTINGS.items():
                cols = [[v] * B for v in w]
                arms[what] = (lambda cols=cols: vn.op_sample_warpers(x, T, ks, seed, ctr, [1.0] * B, [1.0] * B,
                                                                     *cols))
            times = {a: [] for a in arms}
            for r in range(rounds):          # the arms alternate, in reverse order every other round
                for a in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                    times[a].append(time_us(arms[a], iters))
            for a, xs in times.items():
                print(json.dumps(dict(B=B, V=V, top_k=k, setting=a, us_per_call=spread(xs), rounds=rounds, card=name,
                                      power_limit=limit)), flush=True)


def decode(new, reps, name, limit):
    import bench
    from bench_inflight import N_VID, S_MAX, make_model
    for slots in (1, 16):
        model, _, _ = make_model(slots, S_MAX + new)
        ids = bench.synthetic_prompt_ids(seed=1, n_pre=63)[0][None]
        g = torch.Generator(device="cuda").manual_seed(100)
        feats = (torch.randn(1, N_VID, 1024, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
        st = torch.cuda.Stream()
        arms = (("default", {}), ("min_p", dict(min_p=0.05)))
        times = {a: [] for a, _ in arms}

        def run(kw):
            samp = dict(do_sample=True, temperature=0.7, top_k=50, seed=3, **kw)
            st.synchronize()
            t0 = time.perf_counter()
            if slots == 1:
                model.generate(ids, video_spatio_temporal_features=feats, max_new_tokens=new, eos_token_id=None,
                               **samp)
            else:
                reqs = [{"input_ids": ids[0], "video_spatio_temporal_features": feats[0], "seed": 3 + i}
                        for i in range(slots)]
                model.generate_requests(reqs, max_new_tokens=new, eos_token_id=None, slots=slots, **samp)
            st.synchronize()
            return (time.perf_counter() - t0) * 1000.0 / new

        with torch.cuda.stream(st):
            for _, kw in arms:               # warm-up: captures each arm's graphs
                run(kw)
            for r in range(reps):            # the arms alternate, in reverse order every other repetition
                for a, kw in (arms if r % 2 == 0 else arms[::-1]):
                    times[a].append(run(kw))
        for a, xs in times.items():
            print(json.dumps(dict(slots=slots, arm=a, prompt=ids.shape[1], new_tokens=new, ms_per_step=spread(xs),
                                  reps=reps, card=name, power_limit=limit)), flush=True)
        del model
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--skip-decode", action="store_true")
    args = ap.parse_args()
    name, limit = card()
    sampler(args.iters, args.rounds, name, limit)
    if not args.skip_decode:
        decode(args.new, args.reps, name, limit)


if __name__ == "__main__":
    main()

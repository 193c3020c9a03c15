"""The cost of contrastive search (H100; prints one JSON line).

    python tools/bench_contrastive.py [--new 128] [--reps 3] [--out DIR]

Workload: Vicuna-7B shapes with random bf16 weights, B = 1 and B = 4 prompts with video (S = 448: 356 video rows),
EOS off, --new tokens.
(a) ms per generated token of generate(): greedy, and penalty_alpha 0.6 with top_k 4 / 6 / 8 (vcl_llm_contrastive_start
    and one CUDA graph of vcl_llm_contrastive_decode). Median of --reps timed calls after one untimed call that
    captures the graphs.
(b) The share of the contrastive kernels in one top_k 8 call's kernel time (torch.profiler, a run of its own): the
    candidate selection, the rank (max cosines and pick) and the column fork.
(c) vcl_op_contrastive_rank alone at S = 448 context rows, D = 4096: us per launch (CUDA events, 200 launches).
The card's name, power limit and SM clock limit are printed with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "video-llava_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402
import vcl_native as vn  # noqa: E402
from bench_inflight import N_VID, S_MAX, make_model  # noqa: E402
from bench_nucleus import card, time_us  # noqa: E402

KS = (4, 6, 8)
BS = (1, 4)


def clocks():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:   # noqa: BLE001
        return "unknown"


def prompts(B):
    ids = bench.synthetic_prompt_ids(seed=1, n_pre=63)[0][None].repeat(B, 1)
    feats = (torch.randn(B, N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100))
             * 0.5).to(torch.bfloat16)
    return ids, feats


def timed(fn, reps):
    st = torch.cuda.Stream()
    out = []
    with torch.cuda.stream(st):
        fn()                                   # captures the graphs
        for _ in range(reps):
            st.synchronize()
            t0 = time.perf_counter()
            fn()
            st.synchronize()
            out.append(time.perf_counter() - t0)
    return statistics.median(out)


def kernel_share(fn):
    """{name: ms} of the contrastive kernels and the total kernel time of one call, from torch.profiler"""
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn()
        st.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            st.synchronize()
    tot, cs = 0.0, {}
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        tot += t
        for name in ("cs_candidates", "cs_sim", "cs_pick", "cs_fork"):
            if name in e.key:
                cs[name] = cs.get(name, 0.0) + t
    return tot, cs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "clocks_max_sm_and_sm": clocks(),
           "workload": f"7B shapes, random bf16, video, S={S_MAX}, EOS off, {a.new} new tokens, alpha 0.6"}
    print("[bench_contrastive]", res["card"], res["clocks_max_sm_and_sm"], flush=True)
    model, eng, _ = make_model(max(BS) * max(KS), S_MAX + a.new + 8)
    res["ms_per_token"] = {}
    for B in BS:
        ids, feats = prompts(B)
        gen = lambda **kw: model.generate(ids, feats, max_new_tokens=a.new, eos_token_id=None, **kw)   # noqa: E731
        row = {"greedy": round(timed(gen, a.reps) * 1e3 / a.new, 3)}
        for k in KS:
            row[f"k{k}"] = round(timed(lambda: gen(penalty_alpha=0.6, top_k=k), a.reps) * 1e3 / a.new, 3)
        res["ms_per_token"][f"B{B}"] = row
        print("[bench_contrastive] (a)", B, row, flush=True)

    res["kernel_share_k8"] = {}
    for B in BS:
        ids, feats = prompts(B)
        tot, cs = kernel_share(lambda: model.generate(ids, feats, max_new_tokens=a.new, eos_token_id=None,
                                                      penalty_alpha=0.6, top_k=8))
        res["kernel_share_k8"][f"B{B}"] = {"total_kernel_ms": round(tot, 2),
                                          **{n: round(v, 3) for n, v in cs.items()},
                                          "share": round(sum(cs.values()) / tot, 4) if tot > 0 else None}
        print("[bench_contrastive] (b)", B, res["kernel_share_k8"][f"B{B}"], flush=True)

    res["op_rank_us"] = {}
    D = 4096
    for B, k in ((1, 4), (1, 8), (4, 8)):
        ctx = torch.randn(B, S_MAX + 1, D, device="cuda").to(torch.bfloat16)
        hid = torch.randn(B * k, D, device="cuda").to(torch.bfloat16)
        p = torch.rand(B * k, device="cuda")
        tok = torch.zeros(B * k, dtype=torch.int32, device="cuda")
        res["op_rank_us"][f"B{B}_k{k}"] = round(
            time_us(lambda: vn.op_contrastive_rank(ctx, [0] * B, S_MAX, hid, p, tok, 0.6), 200), 2)
    print("[bench_contrastive] (c)", res["op_rank_us"], flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_contrastive.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""Device sampling against the stepwise torch path (H100; prints one JSON line).

    python tools/bench_sampling.py [--rounds 5] [--new 256] [--out DIR]

(a) The reference's setting: Vicuna-7B shapes with random bf16 weights, one clip with video at S = 448,
    generate(do_sample=True, temperature=0.2, top_k=50) with EOS disabled and 256 new tokens: the stepwise torch path
    (no seed), the device sampler (seed=...), and greedy generate (the CUDA-graph floor), alternated round by round;
    the median ms per new token over the rounds (prefill included). The "+stops" arms add what the reference's
    caller always passes, an EOS id and a stopping criterion (here an EOS id no token has and a criterion that reads
    the newest token on the host, like KeywordsStoppingCriteria, and never fires), so the device sampler runs its
    chunked loop with the host-side checks between chunks.
(b) The in-flight workload of bench_inflight.py (64 requests, 16..384 new tokens) sampled at T = 0.2 / top_k 50
    against greedy in flight, at 4 and 16 slots: wall seconds, median of the rounds.
(c) The sampling kernel alone (vcl_op_sample) at B = 1, 4, 16 over V = 32 003 rows: its device time from
    torch.profiler over 100 launches (the entry point's own allocation and host-to-device copy of the row settings
    are not in it); microseconds per launch and the rate of the 4 V B bytes each launch reads.
(d) One in-flight decode chunk (vcl_llm_slot_decode, 4 slots at prompt length, 9 tokens) from its CUDA graph,
    greedy against sampled table entries, alternated: ms per call, median of 30.
The card's name and power limit are printed with the numbers.
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
from bench_inflight import S_MAX, inflight, make_model, make_requests  # noqa: E402
from bench_padded import card  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402


def kernel_us(B, V=32003, iters=100):
    from torch.profiler import ProfilerActivity, profile
    x = (torch.randn(B, V, device="cuda") * 2).bfloat16().float()
    args = ([0.2] * B, [50] * B, list(range(B)), [448] * B)
    vn.op_sample(x, *args)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            vn.op_sample(x, *args)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "sample_kernel" in e.key]
    assert len(ev) == 1 and ev[0].count == iters, [(e.key, e.count) for e in ev]
    total = getattr(ev[0], "device_time_total", None) or ev[0].cuda_time_total
    return total / iters


def chunk_ms(model, eng, reqs, slots=4, calls=30):
    """(d): slot_decode of one 9-token chunk at 4 slots from its graph, greedy / sampled entries alternated"""
    st = torch.cuda.Stream()
    first = torch.zeros(slots, dtype=torch.int32, device="cuda")
    pos = []
    with torch.cuda.stream(st):
        for s in range(slots):
            r = reqs[s]
            vs = torch.tensor([model._video_spans(r["input_ids"][None], eng.NV)[0]], dtype=torch.int32, device="cuda")
            eng.slot_prefill(s, r["input_ids"].cuda(), r["video_spatio_temporal_features"], vs, tok_out=first[s:s + 1])
            pos.append(r["input_ids"].numel())
        times = {"greedy": [], "sampled": []}
        for i in range(calls + 1):
            for name, t in (("greedy", 0.0), ("sampled", 0.2)):
                eng.set_sampling(list(range(slots)), [t] * slots, [50] * slots, list(range(slots)))
                st.synchronize()
                t0 = time.perf_counter()
                eng.slot_decode(first, pos, 9)
                st.synchronize()
                if i > 0:
                    times[name].append((time.perf_counter() - t0) * 1e3)
        eng.set_sampling(list(range(slots)), [0.0] * slots, [0] * slots, [0] * slots)
    return {k: round(statistics.median(v), 3) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--inflight-rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    print("[bench_sampling]", res["card"], flush=True)

    res["kernel_us"] = {}
    for B in (1, 4, 16):
        us = kernel_us(B)
        res["kernel_us"][B] = {"us": round(us, 2), "GB_per_s": round(4 * 32003 * B / us / 1e3, 1)}
    print("[bench_sampling] (c)", res["kernel_us"], flush=True)

    model, eng, _ = make_model(16, S_MAX + 400)
    ids = O.make_prompt_ids(O.LlmCfg(), 356, seed=1).cuda()
    feats = (torch.randn(1, 356, 1024, generator=torch.Generator().manual_seed(2)) * 0.5).half().cuda()
    st = torch.cuda.Stream()
    def never(output_ids, scores=None):
        return int(output_ids[0, -1]) == -5            # reads the newest token on the host, never fires
    stops = dict(eos_token_id=-1, stopping_criteria=[never])
    arms = {
        "stepwise": dict(do_sample=True, temperature=0.2, top_k=50, eos_token_id=None),
        "device": dict(do_sample=True, temperature=0.2, top_k=50, seed=7, eos_token_id=None),
        "greedy": dict(eos_token_id=None),
        "stepwise+stops": dict(do_sample=True, temperature=0.2, top_k=50, **stops),
        "device+stops": dict(do_sample=True, temperature=0.2, top_k=50, seed=7, **stops),
    }
    times = {k: [] for k in arms}
    for r in range(a.rounds + 1):
        for name, kw in arms.items():
            with torch.cuda.stream(st):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = model.generate(ids, video_spatio_temporal_features=feats, max_new_tokens=a.new, **kw)
                st.synchronize()
                dt = time.perf_counter() - t0
            assert out.shape[1] == ids.shape[1] + a.new
            if r > 0:                         # round 0 warms every shape and captures the graphs
                times[name].append(dt * 1e3 / a.new)
    res["ms_per_token"] = {k: round(statistics.median(v), 3) for k, v in times.items()}
    res["ms_per_token_spread"] = {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()}
    print("[bench_sampling] (a)", res["ms_per_token"], res["ms_per_token_spread"], flush=True)

    reqs = make_requests(64, 16, 384)
    res["chunk_ms_4_slots"] = chunk_ms(model, eng, reqs)
    print("[bench_sampling] (d)", res["chunk_ms_4_slots"], flush=True)
    sampled = [dict(r, do_sample=True, temperature=0.2, top_k=50, seed=1000 + i) for i, r in enumerate(reqs)]
    res["inflight_s"] = {}
    for slots in (4, 16):
        wall = {"greedy": [], "sampled": []}
        for _ in range(a.inflight_rounds):
            for name, rs in (("greedy", reqs), ("sampled", sampled)):
                with torch.cuda.stream(st):
                    wall[name].append(inflight(model, rs, slots)[1][0])
        res["inflight_s"][slots] = {k: round(statistics.median(v), 3) for k, v in wall.items()}
    print("[bench_sampling] (b)", res["inflight_s"], flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_sampling.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

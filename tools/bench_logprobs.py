"""The cost of log-probs of generated tokens (H100; prints one JSON line).

    python tools/bench_logprobs.py [--calls 20] [--inflight-rounds 2] [--out DIR]

(a) One in-flight decode chunk (vcl_llm_slot_decode, 9 tokens, every slot at its prompt length) at Vicuna-7B shapes
    with random bf16 weights, at 1, 4, 16 and 64 slots: log-probs off, top_n 0, 5 and 20, each with greedy and with
    T = 0.2 / top_k 50 table entries. The eight arms are alternated call by call; ms per call, median of the calls.
    A greedy arm with log-probs on runs the sampler's graph instead of the arg-max kernels (and, at 1..4 slots,
    without the partial arg-max hand-off).
(b) The in-flight workload of bench_inflight.py (64 requests, 16..384 new tokens, 16 slots), greedy, with log-probs
    off and with logprobs=5 (which adds one read-back copy per decode chunk): requests per second, median of the
    rounds, the two arms alternated.
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

from bench_inflight import S_MAX, make_model, make_requests  # noqa: E402
from bench_padded import card  # noqa: E402

ARMS = [(lp, t) for lp in (-1, 0, 5, 20) for t in (0.0, 0.2)]


def chunk_ms(model, eng, reqs, slot_counts, calls):
    st = torch.cuda.Stream()
    n = max(slot_counts)
    first = torch.zeros(n, dtype=torch.int32, device="cuda")
    pos = []
    res = {}
    with torch.cuda.stream(st):
        for s in range(n):
            r = reqs[s]
            vs = torch.tensor([model._video_spans(r["input_ids"][None], eng.NV)[0]], dtype=torch.int32, device="cuda")
            eng.slot_prefill(s, r["input_ids"].cuda(), r["video_spatio_temporal_features"], vs, tok_out=first[s:s + 1])
            pos.append(r["input_ids"].numel())
        for slots in slot_counts:
            clips = list(range(slots))
            times = {a: [] for a in ARMS}
            for i in range(calls + 1):
                for lp, t in ARMS:
                    eng.set_sampling(clips, [t] * slots, [50] * slots, clips)
                    eng.set_logprobs(clips, [lp] * slots)
                    st.synchronize()
                    t0 = time.perf_counter()
                    eng.slot_decode(first[:slots], pos[:slots], 9)
                    st.synchronize()
                    if i > 0:                 # call 0 captures each graph
                        times[(lp, t)].append((time.perf_counter() - t0) * 1e3)
            res[slots] = {f"{'off' if lp < 0 else f'n{lp}'}_{'greedy' if t == 0 else 'T0.2'}":
                          round(statistics.median(v), 3) for (lp, t), v in times.items()}
            print("[bench_logprobs] (a)", slots, res[slots], flush=True)
        eng.set_sampling(list(range(n)), [0.0] * n, [0] * n, [0] * n)
        eng.set_logprobs(list(range(n)), [-1] * n)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--inflight-rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    print("[bench_logprobs]", res["card"], flush=True)
    model, eng, _ = make_model(64, S_MAX + 400)
    reqs = make_requests(64, 16, 384)
    res["chunk_ms"] = chunk_ms(model, eng, reqs, (1, 4, 16, 64), a.calls)

    st = torch.cuda.Stream()
    rps = {"off": [], "n5": []}
    for _ in range(a.inflight_rounds):
        for name, lp in (("off", None), ("n5", 5)):
            with torch.cuda.stream(st):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model.generate_requests(reqs, eos_token_id=None, slots=16, logprobs=lp)
                st.synchronize()
                rps[name].append(len(reqs) / (time.perf_counter() - t0))
    res["inflight_requests_per_s_16_slots"] = {k: round(statistics.median(v), 3) for k, v in rps.items()}
    res["inflight_requests_per_s_rounds"] = {k: [round(x, 3) for x in v] for k, v in rps.items()}
    print("[bench_logprobs] (b)", res["inflight_requests_per_s_16_slots"], flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_logprobs.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

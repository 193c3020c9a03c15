"""Paged against contiguous KV cache on the reference's own decoding: one arm per process.

    python tools/bench_paged.py --model {7b,13b} --arm {contig,paged} [--requests 256] [--max-new 1024]
                                [--stop-min 32] [--stop-max 512] [--budget-gib G] [--out DIR]

The workload is video_chatgpt_infer's: max_new_tokens 1024, sampling at temperature 0.2 with top-k 50 (seeded on the
device), and prompts of 400..448 tokens with video (bench.synthetic_prompt_ids, random pooled features). Random
weights never produce the stop string, so a per-request stopping criterion fires at a seeded length of --stop-min ..
--stop-max new tokens in its place (the role KeywordsStoppingCriteria plays in the reference). max_seq is 1472
(448 + 1024).

Both arms get the same memory budget for the engine: --budget-gib, by default the free device memory at start less
2 GiB. The engine's fixed bytes (both weight copies, the CLIP-less activations, the decode buffers) are computed
from the shapes and checked against the measured resident memory afterwards.
  contig  the contiguous cache with the most slots (at most 64) whose cache and activations (max_seq rows per slot)
          fit the budget
  paged   64 slots, activations for 64 x 512 rows, and a pool of every 128-column block that fits the rest
Each arm runs generate_requests once as a warm-up over the first 64 requests, then the whole set, timed with a host
clock ended by a stream synchronise. Prints one JSON line: the card name and power limit, slots, kv_blocks,
requests/s, generated tokens/s, the engine's resident memory, and (paged) preemptions, bytes swapped to host memory
and the peak blocks in use.
"""
import argparse
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "video-llava_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402
import vcl_native as vn  # noqa: E402
from bench_padded import card  # noqa: E402
from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM  # noqa: E402

S_MAX, N_VID, MAX_SEQ, V = 448, 356, 1472, 32003
GIB = 2 ** 30


def shapes(model):
    m = bench.MODELS[model]
    return m["hidden"], m["inter"], m["layers"], m["heads"]


def fixed_bytes(model, max_batch):
    """the engine's bytes that do not depend on the cache or the prefill activations: the row-major LLM weights, their
    slot-ordered decode copy, the embedding table, the projector and the per-clip decode buffers (computed)"""
    D, F, L, _ = shapes(model)
    streamed = L * (4 * D * D + 3 * F * D) + V * D
    return 2 * (2 * streamed + V * D + D * 1024 + 2 * max_batch * N_VID * D) + max_batch * (V * 4 + 16 * D * 2) + GIB // 4


def act_row_bytes(model):
    D, F, _, _ = shapes(model)
    return (6 * D + F) * 2 + 8


class StopAt:
    """Fires once the request has n new tokens (stands in for the stop string of KeywordsStoppingCriteria)"""

    def __init__(self, n):
        self.n, self.start = n, None

    def __call__(self, ids, scores=None):
        if self.start is None:
            self.start = ids.shape[1] - 1
        return ids.shape[1] - self.start >= self.n


def make_requests(n, stop_min, stop_max, max_new):
    rnd = random.Random(0)
    reqs = []
    for i in range(n):
        S = rnd.randint(400, S_MAX)
        ids = bench.synthetic_prompt_ids(seed=1 + i, n_pre=63 - (S_MAX - S))[0]
        feats = (torch.randn(N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100 + i))
                 * 0.5).to(torch.bfloat16)
        reqs.append(dict(input_ids=ids, video_spatio_temporal_features=feats, max_new_tokens=max_new,
                         stop=rnd.randint(stop_min, stop_max)))
    return reqs


def with_criteria(reqs):
    return [dict({k: v for k, v in r.items() if k != "stop"}, stopping_criteria=[StopAt(r["stop"])]) for r in reqs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="13b", choices=list(bench.MODELS))
    ap.add_argument("--arm", required=True, choices=["contig", "paged"])
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--max-new", type=int, default=1024)
    ap.add_argument("--stop-min", type=int, default=32)
    ap.add_argument("--stop-max", type=int, default=512)
    ap.add_argument("--budget-gib", type=float, default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.init()
    D, F, L, H = shapes(a.model)
    free0 = torch.cuda.mem_get_info()[0]
    _, llm = bench.device_weights(a.model, "cuda")
    weights_in = sum(t.numel() * t.element_size() for t in llm.values())
    budget = int(a.budget_gib * GIB) if a.budget_gib else free0 - 2 * GIB - weights_in
    col = 2 * L * H * 128 * 2                                  # one cache column of one sequence, K and V
    if a.arm == "contig":
        per_slot = col * MAX_SEQ + MAX_SEQ * act_row_bytes(a.model)
        slots = min(64, (budget - fixed_bytes(a.model, 64)) // per_slot)
        max_batch, kv_blocks = slots, None
    else:
        slots = max_batch = 64
        rest = budget - fixed_bytes(a.model, 64) - 64 * 512 * act_row_bytes(a.model)
        kv_blocks = rest // vn.kv_block_bytes(L, H)
    if slots < 1 or (kv_blocks is not None and kv_blocks < 2):
        raise SystemExit(f"budget {budget / GIB:.1f} GiB leaves no cache")
    cfg = VideoChatGPTConfig(hidden_size=D, intermediate_size=F, num_hidden_layers=L, num_attention_heads=H,
                             vocab_size=V, use_mm_proj=True, mm_hidden_size=1024)
    model = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=int(max_batch), max_seq=MAX_SEQ,
                                         max_slots=int(slots), kv_blocks=None if kv_blocks is None else int(kv_blocks))
    vc = model.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    model.load_state_dict(llm)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    model._ensure_engine(need_llm=True)
    torch.cuda.synchronize()
    resident = free1 - torch.cuda.mem_get_info()[0]
    model._state = {}
    del llm
    torch.cuda.empty_cache()

    reqs = make_requests(a.requests, a.stop_min, a.stop_max, a.max_new)
    kw = dict(eos_token_id=None, do_sample=True, temperature=0.2, top_k=50, seed=1234, packed_admission=True)
    model.generate_requests(with_criteria(reqs[:64]), **kw)            # warm-up: graphs, allocator
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    outs = model.generate_requests(with_criteria(reqs), **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    new = sum(o.shape[1] - r["input_ids"].numel() for o, r in zip(outs, reqs))
    assert all(o.shape[1] - r["input_ids"].numel() == r["stop"] for o, r in zip(outs, reqs))
    name, power = card()
    res = dict(model=a.model, arm=a.arm, card=name, power_limit=power, requests=len(reqs), max_seq=MAX_SEQ,
               slots=int(slots), kv_blocks=kv_blocks and int(kv_blocks), budget_gib=round(budget / GIB, 2),
               resident_gib=round(resident / GIB, 2), wall_s=round(wall, 2), requests_per_s=round(len(reqs) / wall, 3),
               tokens_per_s=round(new / wall, 1), new_tokens=new)
    if kv_blocks:
        st = model.last_kv_stats
        res.update(preemptions=st["preemptions"], swapped_gb=round(st["swapped_bytes"] / 1e9, 2),
                   peak_blocks=st["peak_blocks"])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f"bench_paged_{a.model}_{a.arm}.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

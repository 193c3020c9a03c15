"""Multi-turn video chat served in flight on the paged KV cache: each follow-up re-submitted as a whole new prompt
against conversation sessions ("session" / "continues" in generate_requests).

    python tools/bench_sessions.py [--model 7b] [--conversations 32] [--pools 400,120] [--out DIR]

N conversations x 3 turns. Turn 1 is a video prompt of 400..448 tokens (bench.synthetic_prompt_ids, random pooled
features); every answer stops at a seeded 32..256 new tokens (a per-request stopping criterion in place of the stop
string random weights never produce); follow-ups are 16..48 random text tokens. Sampling at temperature 0.2, top-k 50,
seeded per request. max_seq 2048, 64 slots, packed admission.
  resubmit  turns 2 and 3 re-submit the whole conversation as a new prompt (chunked_prefill=True past 512 tokens)
  sessions  turn 1 starts a session per conversation; turns 2 and 3 continue it, prefilling only the tail
The two arms do NOT return identical tokens: a re-prefilled conversation holds GEMM-written cache columns where a
continued one holds the decode's GEMV-written ones, so the sampled answers drift apart; their lengths (the stopping
criterion) are the same. --pools: one engine per kv_blocks value, e.g. one that holds every kept conversation and one
that forces kept conversations out to host memory. Each arm runs once untimed on the first 4 conversations (graphs,
allocator), then timed turn by turn with a host clock ended by a stream synchronise. Prints one JSON line per pool and
arm: the card and power limit, wall seconds per turn, prefill rows per turn, preemptions, kept-conversation swaps and
bytes.
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
from bench_padded import card  # noqa: E402
from bench_paged import N_VID, S_MAX, V, StopAt, shapes  # noqa: E402
from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM  # noqa: E402

MAX_SEQ, SLOTS, TURNS, MAX_NEW = 2048, 64, 3, 256


def conversations(n):
    """[conv][turn] -> (ids [S] host, feats or None, stop length)"""
    rnd = random.Random(0)
    out = []
    for c in range(n):
        S = rnd.randint(400, S_MAX)
        ids = bench.synthetic_prompt_ids(seed=1 + c, n_pre=63 - (S_MAX - S))[0]
        feats = (torch.randn(N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100 + c))
                 * 0.5).to(torch.bfloat16)
        turns = [(ids, feats, rnd.randint(32, 256))]
        for t in range(1, TURNS):
            k = rnd.randint(16, 48)
            turns.append((torch.randint(3, 32000, (k,), generator=torch.Generator().manual_seed(7000 + 10 * c + t)),
                          None, rnd.randint(32, 256)))
        out.append(turns)
    return out


def run(model, convs, arm):
    """the turns of every conversation; returns per-turn (wall seconds, prefill rows) and the summed kv stats"""
    prev = [None] * len(convs)
    turns, totals = [], dict(preemptions=0, session_swaps=0, session_swapped_bytes=0, swapped_bytes=0)
    for t in range(TURNS):
        reqs, rows = [], 0
        for c, conv in enumerate(convs):
            ids, f, stop = conv[t]
            r = dict(max_new_tokens=MAX_NEW, stopping_criteria=[StopAt(stop)], seed=10 * c + t)
            if f is not None:
                r["video_spatio_temporal_features"] = f
            if arm == "sessions":
                r["input_ids"] = ids
                r["session" if t == 0 else "continues"] = c
                rows += ids.numel() + (t > 0)
            else:
                r["input_ids"] = ids if prev[c] is None else torch.cat([prev[c], ids])
                rows += r["input_ids"].numel()
            reqs.append(r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs = model.generate_requests(reqs, eos_token_id=None, do_sample=True, temperature=0.2, top_k=50,
                                       packed_admission=True, chunked_prefill=True)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        for c, o in enumerate(outs):
            prev[c] = o[0].cpu()
        st = model.last_kv_stats
        for k in totals:
            totals[k] += st[k]
        turns.append(dict(wall_s=round(wall, 3), prefill_rows=rows))
    model.end_session()
    return turns, totals


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="7b", choices=list(bench.MODELS))
    ap.add_argument("--conversations", type=int, default=32)
    ap.add_argument("--pools", default="400,120", help="kv_blocks of each engine, comma-separated")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.init()
    D, F, L, H = shapes(a.model)
    _, llm = bench.device_weights(a.model, "cuda")
    convs = conversations(a.conversations)
    name, power = card()
    lines = []
    for kv_blocks in (int(x) for x in a.pools.split(",")):
        cfg = VideoChatGPTConfig(hidden_size=D, intermediate_size=F, num_hidden_layers=L, num_attention_heads=H,
                                 vocab_size=V, use_mm_proj=True, mm_hidden_size=1024)
        model = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=SLOTS, max_seq=MAX_SEQ, max_slots=SLOTS,
                                             kv_blocks=kv_blocks)
        vc = model.get_model().vision_config
        vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
        model.load_state_dict(llm)
        model._ensure_engine(need_llm=True)
        model._state = {}
        for arm in ("resubmit", "sessions"):
            run(model, convs[:4], arm)                               # warm-up
            turns, totals = run(model, convs, arm)
            res = dict(model=a.model, card=name, power_limit=power, arm=arm, kv_blocks=kv_blocks,
                       conversations=len(convs), slots=SLOTS, turns=turns,
                       total_wall_s=round(sum(t["wall_s"] for t in turns), 3), **totals)
            lines.append(json.dumps(res))
            print(lines[-1], flush=True)
        model._engine.close()
        del model
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f"bench_sessions_{a.model}.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

"""Paged against contiguous KV cache on the reference's own decoding: one arm per process.

    python tools/bench_paged.py --model {7b,13b} --arm {contig,paged} [--requests 256] [--max-new 1024]
                                [--stop-min 32] [--stop-max 512] [--budget-gib G] [--out DIR]
                                [--transcript-tokens LO-HI]

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

--transcript-tokens LO-HI: the --use_asr prompts of the reference's eval scripts. Each prompt gets a transcript of a
seeded LO..HI tokens appended, max_seq is 2048, and max_new_tokens is capped so that the longest prompt fits. The paged
arm then runs generate_requests(chunked_prefill=True) and also reports the chunked prompts and chunk calls. Both arms
then also report the share of the wall time spent in prefill calls (each one timed between two stream synchronises),
and the time of one 1024-token prompt: the contiguous engine's one-shot slot_prefill, or the paged engine's two
512-row chunk calls (median of 10 after a warm-up).
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


def make_requests(n, stop_min, stop_max, max_new, transcript=None):
    rnd = random.Random(0)
    reqs = []
    for i in range(n):
        S = rnd.randint(400, S_MAX)
        ids = bench.synthetic_prompt_ids(seed=1 + i, n_pre=63 - (S_MAX - S))[0]
        if transcript:
            t = rnd.randint(*transcript)
            ids = torch.cat([ids, torch.randint(3, 32000, (t,), generator=torch.Generator().manual_seed(5000 + i))])
        feats = (torch.randn(N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100 + i))
                 * 0.5).to(torch.bfloat16)
        reqs.append(dict(input_ids=ids, video_spatio_temporal_features=feats, max_new_tokens=max_new,
                         stop=rnd.randint(stop_min, stop_max)))
    return reqs


def with_criteria(reqs):
    return [dict({k: v for k, v in r.items() if k != "stop"}, stopping_criteria=[StopAt(r["stop"])]) for r in reqs]


def time_1024(model, paged, reps=10):
    """ms of one 1024-token text prompt into slot 0: one-shot slot_prefill (contiguous) or two 512-row chunk calls
    into a fresh table row (paged), median of reps after a warm-up"""
    eng = model._engine
    ids = torch.randint(3, 32000, (1024,), generator=torch.Generator().manual_seed(7)).to("cuda")
    vs = torch.tensor([vn.NO_VIDEO], dtype=torch.int32, device="cuda")
    if paged:
        table = [[0] * eng.table_row for _ in range(eng.n_slots)]
        table[0][:8] = list(range(1, 9))
        eng.set_block_table(table)

    def once():
        if paged:
            for st in (0, 512):
                eng.slots_prefill_chunk([0], [st], [1024], [ids[st:st + 512]], [None], [0])
        else:
            eng.slot_prefill(0, ids[None], None, vs)
    once()
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        once()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
    if paged:
        eng.set_block_table([[0] * eng.table_row for _ in range(eng.n_slots)])
    return sorted(times)[reps // 2]


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
    ap.add_argument("--transcript-tokens", default=None, metavar="LO-HI")
    a = ap.parse_args()
    transcript = tuple(int(x) for x in a.transcript_tokens.split("-")) if a.transcript_tokens else None
    max_seq = 2048 if transcript else MAX_SEQ
    if transcript:
        a.max_new = min(a.max_new, max_seq - S_MAX - transcript[1])
        a.stop_max = min(a.stop_max, a.max_new)
        a.stop_min = min(a.stop_min, a.stop_max)
    torch.cuda.init()
    D, F, L, H = shapes(a.model)
    free0 = torch.cuda.mem_get_info()[0]
    _, llm = bench.device_weights(a.model, "cuda")
    weights_in = sum(t.numel() * t.element_size() for t in llm.values())
    budget = int(a.budget_gib * GIB) if a.budget_gib else free0 - 2 * GIB - weights_in
    col = 2 * L * H * 128 * 2                                  # one cache column of one sequence, K and V
    if a.arm == "contig":
        per_slot = col * max_seq + max_seq * act_row_bytes(a.model)
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
    model = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=int(max_batch), max_seq=max_seq,
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

    reqs = make_requests(a.requests, a.stop_min, a.stop_max, a.max_new, transcript)
    kw = dict(eos_token_id=None, do_sample=True, temperature=0.2, top_k=50, seed=1234, packed_admission=True)
    if transcript and kv_blocks:
        kw["chunked_prefill"] = True
    model.generate_requests(with_criteria(reqs[:64]), **kw)            # warm-up: graphs, allocator
    torch.cuda.synchronize()
    eng = model._engine
    prefill_s = [0.0]
    if transcript:                                   # time every prefill call between two stream synchronises
        for name in ("slot_prefill", "slots_prefill", "slots_prefill_chunk"):
            def timed(*args, _f=getattr(eng, name), **kwargs):
                torch.cuda.synchronize()
                t = time.perf_counter()
                r = _f(*args, **kwargs)
                torch.cuda.synchronize()
                prefill_s[0] += time.perf_counter() - t
                return r
            setattr(eng, name, timed)
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
                   peak_blocks=st["peak_blocks"], chunked_prefills=st["chunked_prefills"],
                   chunk_calls=st["chunk_calls"])
    if transcript:
        res.update(transcript_tokens=a.transcript_tokens, max_new=a.max_new,
                   prefill_share=round(prefill_s[0] / wall, 3), prompt_1024_ms=round(time_1024(model, kv_blocks), 2))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f"bench_paged_{a.model}_{a.arm}.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

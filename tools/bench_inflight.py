"""In-flight (continuous) batching against static batches and one request at a time.

    python tools/bench_inflight.py [--requests 64] [--min-new 16] [--max-new 384] [--slots 4,8,16]
                                   [--chunks 16] [--repeats 2] [--no-static] [--no-alone] [--out DIR]
                                   [--llm-weight-format {bf16,fp8_e4m3}]
    python tools/bench_inflight.py --prefill-cost [--ks 1,2,4,8,16] [--iters 10] [--out DIR]

More than 16 slots set max_slots on the engine (one slot per clip of max_batch = the largest slot count); the
engine's resident memory (free device memory before and after creating and loading it) is reported.
Vicuna-7B shapes with random-init bf16 weights (bench.device_weights, seed 0), random pooled video features, and
prompts of 400..448 tokens (bench.synthetic_prompt_ids with a shorter text before the video). Random weights never
produce a real EOS, so each request's seeded max_new_tokens (uniform over --min-new .. --max-new) stands in for
one, and every arm produces the same tokens per request. Arms, per slot count:
  (a) static    consecutive groups of `slots` requests, each one left-padded generate (attention_mask) that runs
                to the group's longest request; the outputs are cut to each request's length
  (b) inflight  generate_requests with the same slots (and each chunk length of --chunks, set on the class
                constant _SLOT_CHUNK)
  (p) packed    (b) with packed_admission=True: every admission point fills all free slots with one packed
                prefill (vcl_llm_slots_prefill)
  (c) alone     one generate per request; run once, after the others (it is the longest and does not depend on
                the slot count)
After one warm-up round of (a), (b) and (p) over the first `slots` requests, they alternate --repeats times.
Each arm is timed with a host clock around its calls, ended by a stream synchronise. The admission share of (b) and
(p) is the device time of their prefills (CUDA events around each call) over the wall time.
--prefill-cost instead times admission alone: one slots_prefill of k requests (400..448 tokens with video) against
k slot_prefill calls of the same requests, for each k of --ks, the two arms alternated, CUDA events around each
arm, median and spread over --iters rounds after one warm-up.
Prints one JSON line: per arm requests/s, generated tokens/s, median and p90 request latency (from the start of
the arm to the synchronise after the call that completed the request: for (a) its group, for (b) the whole run,
since generate_requests returns once), the card name and power limit, and whether every request's tokens agree
across the arms under the margin rule of the parity tests (identical up to the first step where the request's
own top-1/top-2 logit margin is below 3 bf16 ulps).
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "video-llava_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402
from bench_padded import card  # noqa: E402
from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM  # noqa: E402

S_MAX, N_VID = 448, 356


def make_model(max_batch, max_seq, weight_format="bf16"):
    """the engine has max_batch cache slots (max_slots above 16); returns (model, engine, resident bytes: free device
    memory before creating the engine minus after loading it)"""
    m = bench.MODELS["7b"]
    cfg = VideoChatGPTConfig(hidden_size=m["hidden"], intermediate_size=m["inter"], num_hidden_layers=m["layers"],
                             num_attention_heads=m["heads"], vocab_size=32003, use_mm_proj=True, mm_hidden_size=1024)
    model = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=max_batch, max_seq=max_seq,
                                         max_slots=max_batch if max_batch > 16 else None,
                                         llm_weight_format=weight_format)
    vc = model.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    _, llm = bench.device_weights("7b", "cuda")
    model.load_state_dict(llm)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    eng = model._ensure_engine(need_llm=True)
    torch.cuda.synchronize()
    resident = free0 - torch.cuda.mem_get_info()[0]
    model._state = {}
    del llm
    torch.cuda.empty_cache()
    return model, eng, resident


def make_requests(n, min_new, max_new, min_len=400):
    rnd = random.Random(0)
    reqs = []
    for i in range(n):
        S = rnd.randint(min_len, S_MAX)
        ids = bench.synthetic_prompt_ids(seed=1 + i, n_pre=63 - (S_MAX - S))[0]
        feats = (torch.randn(N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100 + i))
                 * 0.5).to(torch.bfloat16)
        reqs.append(dict(input_ids=ids, video_spatio_temporal_features=feats,
                         max_new_tokens=rnd.randint(min_new, max_new)))
    return reqs


def static(model, reqs, slots):
    """-> (new tokens per request, completion time per request in s from the start)"""
    toks, done, t0 = [], [], time.perf_counter()
    for g in range(0, len(reqs), slots):
        grp = reqs[g:g + slots]
        S = max(r["input_ids"].numel() for r in grp)
        ids = torch.zeros(len(grp), S, dtype=torch.int64)
        mask = torch.zeros(len(grp), S, dtype=torch.int64)
        for b, r in enumerate(grp):
            n = r["input_ids"].numel()
            ids[b, S - n:], mask[b, S - n:] = r["input_ids"], 1
        feats = torch.stack([r["video_spatio_temporal_features"] for r in grp])
        out = model.generate(ids, video_spatio_temporal_features=feats, attention_mask=mask, eos_token_id=None,
                             max_new_tokens=max(r["max_new_tokens"] for r in grp))
        out = out[:, S:].tolist()
        torch.cuda.current_stream().synchronize()
        t = time.perf_counter() - t0
        for b, r in enumerate(grp):
            toks.append(out[b][:r["max_new_tokens"]])
            done.append(t)
    return toks, done


def inflight(model, reqs, slots, packed=False):
    t0 = time.perf_counter()
    outs = model.generate_requests(reqs, eos_token_id=None, slots=slots, packed_admission=packed)
    torch.cuda.current_stream().synchronize()
    t = time.perf_counter() - t0
    return [o[0, r["input_ids"].numel():].tolist() for o, r in zip(outs, reqs)], [t] * len(reqs)


def alone(model, reqs):
    toks, done, t0 = [], [], time.perf_counter()
    for r in reqs:
        out = model.generate(r["input_ids"][None], video_spatio_temporal_features=r["video_spatio_temporal_features"][None],
                             eos_token_id=None, max_new_tokens=r["max_new_tokens"])
        toks.append(out[0, r["input_ids"].numel():].tolist())
        torch.cuda.current_stream().synchronize()
        done.append(time.perf_counter() - t0)
    return toks, done


def summary(wall, done, n_tokens):
    lat = sorted(done)
    return {"wall_s": round(wall, 3), "requests_per_s": round(len(done) / wall, 3),
            "tokens_per_s": round(n_tokens / wall, 1), "latency_median_s": round(statistics.median(lat), 3),
            "latency_p90_s": round(lat[min(len(lat) - 1, int(0.9 * len(lat)))], 3)}


def agree_to_tie(model, eng, r, a, b):
    """a, b: two token lists of request r. True if they are identical, or first differ at a step where the
    request's own top-1/top-2 logit margin (its prompt + the common prefix, prefilled alone) is below 3 ulps."""
    d = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), None)
    if d is None:
        return len(a) == len(b)
    ids = torch.cat([r["input_ids"], torch.tensor(a[:d], dtype=torch.int64)])[None].cuda()
    vs = model._spans_dev(ids, r["video_spatio_temporal_features"], eng.NV)
    _, lg, _ = eng.prefill(ids, r["video_spatio_temporal_features"][None], vs, want_logits=True, want_token=False)
    top = torch.topk(lg[0], 2).values
    ulp = top[0].abs().clamp_min(2 ** -6) * 2 ** -7
    return bool(((top[0] - top[1]) / ulp) < 3)


def prefill_cost(model, eng, reqs, ks, iters):
    """-> {k: {"packed_ms": median, "single_ms": median, "..._range": [min, max]}} over iters alternated rounds"""
    res = {}
    for k in ks:
        grp = reqs[:k]
        ids = [r["input_ids"].cuda() for r in grp]
        feats = [r["video_spatio_temporal_features"] for r in grp]
        vstarts = [int(model._video_spans(r["input_ids"][None], eng.NV)[0]) for r in grp]
        tok = torch.empty(k, dtype=torch.int32, device="cuda")

        def single():
            for s in range(k):
                vs = torch.tensor([vstarts[s]], dtype=torch.int32, device="cuda")
                eng.slot_prefill(s, ids[s][None], feats[s], vs, tok_out=tok[s:s + 1])

        def packed():
            eng.slots_prefill(list(range(k)), ids, feats, vstarts, tok_out=tok)

        times = {"single": [], "packed": []}
        for it in range(iters + 1):
            for name, fn in (("single", single), ("packed", packed)) if it % 2 == 0 else (("packed", packed),
                                                                                           ("single", single)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                if it > 0:
                    times[name].append(e0.elapsed_time(e1))
        res[k] = {}
        for name, t in times.items():
            res[k][f"{name}_ms"] = round(statistics.median(t), 2)
            res[k][f"{name}_range_ms"] = [round(min(t), 2), round(max(t), 2)]
        res[k]["speedup"] = round(res[k]["single_ms"] / res[k]["packed_ms"], 3)
        log(f"prefill k={k}: {res[k]}")
    return res


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--min-new", type=int, default=16)
    ap.add_argument("--max-new", type=int, default=384)
    ap.add_argument("--slots", default="4,8,16")
    ap.add_argument("--chunks", default=None, help="chunk lengths of the in-flight arm (default: the class constant)")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--no-alone", action="store_true", help="skip arm (c)")
    ap.add_argument("--no-static", action="store_true", help="skip arm (a)")
    ap.add_argument("--prefill-cost", action="store_true", help="time admission alone (see above)")
    ap.add_argument("--ks", default="1,2,4,8,16")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/bench_inflight.json")
    ap.add_argument("--llm-weight-format", default="bf16", choices=["bf16", "fp8_e4m3"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_inflight.py needs an H100 (no CPU measurement)")
    name, power = card()
    slot_counts = [int(s) for s in a.slots.split(",")]
    default_chunk = VideoChatGPTLlamaForCausalLM._SLOT_CHUNK
    chunks = [int(c) for c in a.chunks.split(",")] if a.chunks else [default_chunk]
    if a.prefill_cost:
        ks = [int(k) for k in a.ks.split(",")]
        model, eng, _ = make_model(max(ks), S_MAX + a.max_new, a.llm_weight_format)
        reqs = make_requests(max(ks), a.min_new, a.max_new)
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            res = {"what": "one slots_prefill of k requests against k slot_prefill calls, prompts 400..448 tokens "
                           "with video, Vicuna-7B shapes, CUDA events, median of alternated rounds",
                   "card": name, "power_limit": power, "iters": a.iters,
                   "prefill": prefill_cost(model, eng, reqs, ks, a.iters)}
        st.synchronize()
        line = json.dumps(res)
        print(line)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "bench_prefill_cost.json"), "w") as f:
                f.write(line + "\n")
        return
    model, eng, resident = make_model(max(slot_counts), S_MAX + a.max_new, a.llm_weight_format)
    reqs = make_requests(a.requests, a.min_new, a.max_new)
    n_tokens = sum(r["max_new_tokens"] for r in reqs)
    # admissions: device time of every slot prefill of the in-flight arm
    prefill_ms = []
    slot_prefill = eng.slot_prefill

    def timed_prefill(*args, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = slot_prefill(*args, **kw)
        e1.record()
        prefill_ms.append((e0, e1))
        return out

    eng.slot_prefill = timed_prefill
    slots_prefill = eng.slots_prefill

    def timed_slots_prefill(*args, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = slots_prefill(*args, **kw)
        e1.record()
        prefill_ms.append((e0, e1))
        return out

    eng.slots_prefill = timed_slots_prefill
    st = torch.cuda.Stream()          # decode loops are captured into CUDA graphs on a non-default stream
    res = {"what": f"{a.requests} requests, prompts 400..{S_MAX} tokens with video, max_new_tokens uniform "
                   f"{a.min_new}..{a.max_new} ({n_tokens} tokens), Vicuna-7B shapes, random bf16 weights",
           "card": name, "power_limit": power, "repeats": a.repeats, "llm_weight_format": a.llm_weight_format,
           "resident_gib": round(resident / 2 ** 30, 2), "max_seq": S_MAX + a.max_new, "arms": {}}
    tokens = {}
    with torch.cuda.stream(st):
        for slots in slot_counts:
            warm = reqs[:slots]
            if not a.no_static:
                static(model, warm, slots)
            for c in chunks:
                VideoChatGPTLlamaForCausalLM._SLOT_CHUNK = c
                inflight(model, warm, slots)
                inflight(model, warm, slots, packed=True)
            runs = {}
            for rep in range(a.repeats):
                if not a.no_static:
                    t0 = time.perf_counter()
                    tok, done = static(model, reqs, slots)
                    runs.setdefault("static", []).append((time.perf_counter() - t0, done))
                    log(f"slots {slots} static {runs['static'][-1][0]:.2f} s")
                    tokens[f"static_{slots}"] = tok
                for c in chunks:
                    VideoChatGPTLlamaForCausalLM._SLOT_CHUNK = c
                    for packed in ((False, True) if rep % 2 == 0 else (True, False)):
                        arm = f"{'packed' if packed else 'inflight'}_chunk{c}"
                        prefill_ms.clear()
                        t0 = time.perf_counter()
                        tok, done = inflight(model, reqs, slots, packed=packed)
                        wall = time.perf_counter() - t0
                        adm = sum(e0.elapsed_time(e1) for e0, e1 in prefill_ms) / 1e3
                        runs.setdefault(arm, []).append((wall, done, adm, len(prefill_ms)))
                        log(f"slots {slots} {arm} {wall:.2f} s, admissions {adm:.2f} s in {len(prefill_ms)} calls")
                        tokens[f"{arm}_{slots}"] = tok
            for arm, rs in runs.items():
                best = min(rs, key=lambda x: x[0])
                s = summary(best[0], best[1], n_tokens)
                s["wall_s_all"] = [round(x[0], 3) for x in rs]
                if arm.startswith(("inflight", "packed")):
                    s["admission_share"] = round(best[2] / best[0], 3)
                    s["admission_calls"] = best[3]
                res["arms"][f"{arm}_slots{slots}"] = s
        VideoChatGPTLlamaForCausalLM._SLOT_CHUNK = default_chunk
        if not a.no_alone:
            t0 = time.perf_counter()
            tok, done = alone(model, reqs)
            res["arms"]["alone"] = summary(time.perf_counter() - t0, done, n_tokens)
            log(f"alone {res['arms']['alone']['wall_s']} s")
            tokens["alone"] = tok
        # agreement: every arm against the first one, per request
        names = list(tokens)
        ref = tokens[names[0]]
        identical = to_tie = 0
        for i, r in enumerate(reqs):
            same = all(tokens[k][i] == ref[i] for k in names)
            identical += same
            to_tie += same or all(agree_to_tie(model, eng, r, ref[i], tokens[k][i]) for k in names)
    st.synchronize()
    res["tokens_identical_across_arms"] = f"{identical}/{len(reqs)}"
    # packed admission against one at a time with the same slots and chunk: bit-identical by construction
    for slots in slot_counts:
        for c in chunks:
            a_tok, p_tok = tokens[f"inflight_chunk{c}_{slots}"], tokens[f"packed_chunk{c}_{slots}"]
            res[f"packed_identical_to_inflight_slots{slots}_chunk{c}"] = \
                f"{sum(x == y for x, y in zip(a_tok, p_tok))}/{len(reqs)}"
    res["tokens_match_margin_rule"] = f"{to_tie}/{len(reqs)}"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_inflight.json"), "w") as f:
            f.write(line + "\n")
    if to_tie != len(reqs):
        raise SystemExit("a request's tokens differ across arms before a near-tie")


if __name__ == "__main__":
    main()

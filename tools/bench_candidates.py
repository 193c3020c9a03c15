"""Multiple-choice scoring: score_candidates (one prefill per prompt, forked cache slots, one packed continuation of
the options) against scoring every prompt + option sequence with forward(labels=...).

    python tools/bench_candidates.py [--repeats 5] [--warmup 1] [--out DIR]

Vicuna-7B shapes with random-init bf16 weights (bench.device_weights, seed 0) and random video features; the vision
tower is not part of the measurement. A question is a prompt of 400 .. 448 tokens with video (bench.synthetic_prompt_ids
with a shorter preamble) and 5 seeded options of 4 .. 32 tokens. Workloads of 1 and 16 questions; one model (max_batch
16, max_seq 480, 16 slots) serves every arm:
  candidates   score_candidates
  padded       forward(labels=...) over left-padded batches of up to 16 prompt + option sequences, then the option
               rows' log-softmax gathered from the returned logits
  per_option   the same, one sequence per forward
The arms alternate, `--repeats` times after `--warmup` rounds, each timed with a host clock around the call ended by a
synchronise; the JSON line reports the median ms per question. One more score_candidates run records CUDA events
around each engine call: the prompt prefills, the forks and the packed continuations. The largest difference between
arms in an option's summed log-prob is reported too. The card's name and power limit are read in the same run.
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
from bench_padded import card  # noqa: E402

N_OPT, BATCH = 5, 16


def make_model():
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    m = bench.MODELS["7b"]
    cfg = VideoChatGPTConfig(hidden_size=m["hidden"], intermediate_size=m["inter"], num_hidden_layers=m["layers"],
                             num_attention_heads=m["heads"], vocab_size=32003, use_mm_proj=True, mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    model = VideoChatGPTLlamaForCausalLM(cfg, clip_config=clip, max_batch=BATCH, max_seq=480, max_slots=BATCH)
    vc = model.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    clip_w, llm = bench.device_weights("7b", "cuda")
    del clip_w
    model.load_state_dict(llm, strict=False)
    model._ensure_engine(need_llm=True)
    return model


def questions(n, seed=0):
    out = []
    for i in range(n):
        g = torch.Generator().manual_seed(seed * 1000 + i)
        S = 400 + int(torch.randint(0, 49, (1,), generator=g))
        ids = bench.synthetic_prompt_ids(seed=1 + i, n_pre=63 - (448 - S))[0]
        opts = [torch.randint(3, 32000, (int(torch.randint(4, 33, (1,), generator=g)),), generator=g)
                for _ in range(N_OPT)]
        f = (torch.randn(356, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(i)) * 0.5)
        out.append((ids, opts, f.to(torch.bfloat16)))
    return out


def by_forward(m, qs, batch):
    """summed option log-probs [n_q][N_OPT] (float64) from forward(labels=...) over batches of `batch` sequences"""
    seqs = [(b, j, torch.cat([ids, c]), ids.numel(), c, f) for b, (ids, opts, f) in enumerate(qs)
            for j, c in enumerate(opts)]
    out = [[0.0] * N_OPT for _ in qs]
    for i in range(0, len(seqs), batch):
        grp = seqs[i:i + batch]
        S = max(s[2].numel() for s in grp)
        ids = torch.zeros(len(grp), S, dtype=torch.int64)
        mask = torch.zeros(len(grp), S, dtype=torch.int64)
        lab = torch.full((len(grp), S), -100, dtype=torch.int64)
        for r, (_, _, x, P, c, _) in enumerate(grp):
            ids[r, S - x.numel():] = x
            mask[r, S - x.numel():] = 1
            lab[r, S - c.numel():] = c
        feats = torch.stack([s[5] for s in grp])
        o = m.forward(ids.cuda(), attention_mask=mask.cuda(), labels=lab.cuda(), video_spatio_temporal_features=feats)
        for r, (b, j, x, P, c, _) in enumerate(grp):
            rows = o.logits[r, S - c.numel() - 1:S - 1].float()
            out[b][j] = torch.log_softmax(rows, -1)[torch.arange(c.numel()), c.cuda()].double().sum()
    return [[float(v) for v in row] for row in out]


def split(m, qs):
    """CUDA-event time of each kind of engine call inside one score_candidates run"""
    eng = m._engine
    ev = {k: [] for k in ("prefill", "fork", "continuation")}
    orig = {}
    for name, kind in (("slots_prefill", "prefill"), ("slot_prefill", "prefill"), ("slots_fork", "fork"),
                       ("slots_score_append", "continuation")):
        fn = getattr(eng, name)
        orig[name] = fn

        def wrapped(*a, _fn=fn, _kind=kind, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = _fn(*a, **k)
            e1.record()
            ev[_kind].append((e0, e1))
            return r
        setattr(eng, name, wrapped)
    try:
        m.score_candidates([q[0] for q in qs], [q[1] for q in qs], video_spatio_temporal_features=[q[2] for q in qs])
        torch.cuda.synchronize()
    finally:
        for name, fn in orig.items():
            setattr(eng, name, fn)
    return {k: round(sum(a.elapsed_time(b) for a, b in v) / len(qs), 3) for k, v in ev.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/bench_candidates.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_candidates.py needs an H100 (no CPU measurement)")
    name, power = card()
    m = make_model()
    res = {"what": "Vicuna-7B shapes, random bf16 weights, prompts of 400..448 tokens with video, 5 options of 4..32 "
                   "tokens", "card": name, "power_limit": power, "repeats": a.repeats, "warmup": a.warmup}

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    with torch.no_grad():
        for n in (1, 16):
            qs = questions(n)
            arms = {
                "candidates": lambda: [[float(v) for v in o["logprob"]] for o in m.score_candidates(
                    [q[0] for q in qs], [q[1] for q in qs], video_spatio_temporal_features=[q[2] for q in qs])],
                "padded": lambda: by_forward(m, qs, BATCH),
                "per_option": lambda: by_forward(m, qs, 1),
            }
            times = {k: [] for k in arms}
            sums = {}
            for i in range(a.warmup + a.repeats):
                for k, fn in arms.items():
                    t, out = timed(fn)
                    if i >= a.warmup:
                        times[k].append(t / n)
                    sums[k] = out
            diff = max(abs(sums[x][b][j] - sums["candidates"][b][j]) for x in ("padded", "per_option")
                       for b in range(n) for j in range(N_OPT))
            med = {k: round(statistics.median(v), 2) for k, v in times.items()}
            res[f"questions_{n}"] = {
                "ms_per_question": med,
                "speedup_vs_padded": round(med["padded"] / med["candidates"], 2),
                "speedup_vs_per_option": round(med["per_option"] / med["candidates"], 2),
                "candidates_split_ms_per_question": split(m, qs),
                "max_abs_diff_summed_logprob": round(diff, 4),
            }
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_candidates.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

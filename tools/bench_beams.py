"""The cost of beam search (H100; prints one JSON line).

    python tools/bench_beams.py [--new 256] [--baseline-steps 32] [--out DIR]

Workload: Vicuna-7B shapes with random bf16 weights, one clip with video (S = 448: 356 video rows), EOS off,
--new tokens.
(a) ms per generated token of generate(): greedy, and num_beams 2 / 4 / 8 through the device loop (vcl_llm_beam_start
    and CUDA-graph chunks of vcl_llm_beam_decode, the host replaying steps 4-6 between chunks).
(b) num_beams 4 at chunk lengths 4 / 8 / 16 / 32 (the choice of _BEAM_CHUNK).
(c) The same beams through a stepwise host loop, an UPPER BOUND of a host-driven baseline: eager decode_step of the k
    rows, torch log_softmax / topk / gathers on the device, and the reorder as index_select of every layer's K and V.
    The C ABI only copies a whole layer's cache out and back (vcl_kv_cache_copy), so each step moves max_batch clips
    three times where HF's reorder_cache reads and writes k clips once. Two untimed warm-up steps, then
    --baseline-steps steps, ms per step.
(d) Forks: the clip columns the device copied per step in a num_beams 4 / 8 run (counted from the records), times the
    bytes of a column (L * 2 * D * 2).
(e) vcl_op_beam_select alone: us per launch (CUDA events, 200 launches) at B * k = 4 / 16 / 64, V = 32003.
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

import bench  # noqa: E402
import vcl_native as vn  # noqa: E402
from bench_inflight import N_VID, S_MAX, make_model  # noqa: E402
from bench_nucleus import card, time_us  # noqa: E402


def prompt():
    ids = bench.synthetic_prompt_ids(seed=1, n_pre=63)[0][None]
    feats = (torch.randn(1, N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(100))
             * 0.5).to(torch.bfloat16)
    return ids, feats


def timed(fn, reps=2):
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


def forks_per_step(rec, picks, k):
    """columns copied per step: (after step 0) every pick whose parent already had a child"""
    _, beam, _ = vn.beam_records(rec)
    out = []
    for t in range(1, rec.shape[0]):
        par = [int(beam[t, 0, int(picks[t, 0, r])]) for r in range(k)]
        out.append((k - len(set(par))) * t)   # each fork copies columns S .. S + t - 1
    return out


def baseline_ms(model, eng, ids, feats, k, steps):
    """stepwise host loop: eager decode_step over k rows + torch selection + index_select of the whole cache"""
    L = model.config.num_hidden_layers
    S = ids.shape[1]
    vs = torch.tensor([model._video_spans(ids, eng.NV)[0]] * k, dtype=torch.int32, device="cuda")
    rids = ids.cuda().repeat(k, 1)
    _, lg, _ = eng.prefill(rids, feats.repeat(k, 1, 1), vs, want_logits=True, want_token=False)
    scores = torch.zeros(k, device="cuda")
    scores[1:] = -1e9
    V = lg.shape[1]
    for t in range(steps + 2):
        if t == 2:                       # two warm-up steps
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        acc = (torch.log_softmax(lg, dim=-1) + scores[:, None]).reshape(-1)
        top, idx = torch.topk(acc, 2 * k)
        pick = torch.topk(top, k)[1]
        scores, parent, tok = top[pick], idx[pick] // V, (idx[pick] % V).to(torch.int32)
        for layer in range(L):
            kk, vv = eng.kv_cache(layer)
            kk[:k] = kk[:k].index_select(0, parent)
            vv[:k] = vv[:k].index_select(0, parent)
            eng.set_kv_cache(layer, kk, vv)
        lg, _ = eng.decode_step(tok.contiguous(), S + t, want_logits=True)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--baseline-steps", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "workload": f"7B shapes, random bf16, 1 clip, S={S_MAX}, EOS off, {a.new} new tokens"}
    print("[bench_beams]", res["card"], flush=True)
    model, eng, _ = make_model(8, S_MAX + a.new + 8)
    ids, feats = prompt()
    gen = lambda **kw: model.generate(ids, feats, max_new_tokens=a.new, eos_token_id=None, **kw)   # noqa: E731

    res["ms_per_token"] = {"greedy": round(timed(gen) * 1e3 / a.new, 3)}
    for k in (2, 4, 8):
        res["ms_per_token"][f"beams{k}"] = round(timed(lambda: gen(num_beams=k)) * 1e3 / a.new, 3)
        print("[bench_beams] (a)", res["ms_per_token"], flush=True)
    res["beams4_ms_per_token_by_chunk"] = {}
    for c in (4, 8, 16, 32):
        model._BEAM_CHUNK = c
        res["beams4_ms_per_token_by_chunk"][c] = round(timed(lambda: gen(num_beams=4)) * 1e3 / a.new, 3)
        print("[bench_beams] (b)", res["beams4_ms_per_token_by_chunk"], flush=True)
    model._BEAM_CHUNK = type(model)._BEAM_CHUNK

    D, L = model.config.hidden_size, model.config.num_hidden_layers
    col = L * 2 * D * 2
    res["fork"] = {"bytes_per_column": col}
    st = torch.cuda.Stream()
    for k in (4, 8):
        with torch.cuda.stream(st):
            vs = torch.tensor([model._video_spans(ids, eng.NV)[0]], dtype=torch.int32, device="cuda")
            rec, picks = eng.beam_start(ids.cuda(), feats, vs, k, a.new)
            r2, p2 = eng.beam_decode(a.new - 1)
        st.synchronize()
        cols = forks_per_step(torch.cat([rec, r2]).cpu(), torch.cat([picks, p2]).cpu(), k)
        res["fork"][f"beams{k}"] = {"mean_MB_per_step": round(statistics.mean(cols) * col / 2 ** 20, 2),
                                   "max_MB_per_step": round(max(cols) * col / 2 ** 20, 2),
                                   "bound_MB_last_step": round((k - 1) * a.new * col / 2 ** 20, 1)}
    print("[bench_beams] (d)", res["fork"], flush=True)

    res["baseline_host_loop_ms_per_step_upper_bound"] = {}
    for k in (2, 4, 8):
        res["baseline_host_loop_ms_per_step_upper_bound"][f"beams{k}"] = round(
            baseline_ms(model, eng, ids, feats, k, a.baseline_steps), 3)
        print("[bench_beams] (c)", res["baseline_host_loop_ms_per_step_upper_bound"], flush=True)

    res["op_beam_select_us"] = {}
    V = 32003
    for Bk in (4, 16, 64):
        k = 4
        x = (torch.randn(Bk, V, device="cuda") * 3).bfloat16().float()
        sc = -torch.rand(Bk, device="cuda")
        res["op_beam_select_us"][Bk] = round(time_us(lambda: vn.op_beam_select(x, sc, k), 200), 2)
    print("[bench_beams] (e)", res["op_beam_select_us"], flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_beams.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

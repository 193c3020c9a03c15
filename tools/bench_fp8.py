"""bf16 against fp8 (E4M3) LLM weights (H100; prints one JSON line).

    python tools/bench_fp8.py [--rounds 10] [--skip-13b] [--batches 1,4,16] [--decode-only --formats bf16]

(a) 7B decode: Vicuna-7B shapes with random bf16 weights (bench.py's), prompts of S = 448 with video, the CUDA-graph
    decode loop of 31 steps (vcl_llm_decode_loop, 32 tokens) at B = 1, 4 and 16 clips. The bf16 and the fp8 engine
    are both resident and alternate call by call; ms per step is the median over the rounds, and the algorithmic
    rate counts the streamed weight bytes (bf16 slots, or fp8 codes + row scales) plus the KV cache read per step.
(b) One clip with video through the language model (prefill at S = 448 + 32 greedy tokens, EOS off), clips/s of
    both engines, alternated, median; the vision tower is not part of it.
(c) Report only: W~ relative error over the streamed matrices, and on the same prompts the fp8 engine's prefill
    logits against the bf16 engine's on W (relative error) and the greedy agreement of the 32 tokens. The weights
    are random: this says nothing about answer quality on a trained checkpoint.
(d) 13B (one engine at a time): resident memory of the bf16 and the fp8 engine (free device memory before and
    after creating and loading it), and the fp8 decode at B = 4.
--batches: the clip counts of (a); above 16 they run the 17..64-clip ring kernel. --decode-only runs (a) alone, with
the engines of --formats (one engine each; a 7B engine sized for 64 clips holds 16 GB of KV cache, so at 64 clips
run one format per call). --compare-lib PATH (with --decode-only) also creates, for every format, an engine from another
build of libvcl.so (e.g. the parent commit's, built side by side) and alternates the two call by call; --layers N
shortens the model so that both engines fit on one card (the ratio of the two is what this compares).
"tokens_equal" at each B says whether the engines' first tokens and decode_loop tokens of the last round are equal
(for two builds of the same format: an identity check; bf16 against fp8 on the same W need not agree).
The card's name and power limit are printed with the numbers.
"""
import argparse
import gc
import importlib.util
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "video-llava_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import bench  # noqa: E402
import vcl_native as vn  # noqa: E402
import _fp8_ref as R  # noqa: E402
from bench_padded import card  # noqa: E402

S, N_NEW, N_VID = 448, 32, 356


def other_binding(lib_path):
    """a second instance of the vcl_native module bound to another libvcl.so (same C ABI)"""
    spec = importlib.util.spec_from_file_location("vcl_native_other", vn.__file__)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.LIB_PATH = os.path.abspath(lib_path)
    return mod


def engine(model, fmt, max_batch=16, llm=None, binding=None):
    m = bench.MODELS[model]
    c = (binding or vn).vcl_config()
    c.clip_layers, c.clip_hidden, c.clip_inter, c.clip_heads = 0, 1024, 4096, 16
    c.image_size, c.patch_size, c.clip_ln_eps = 224, 14, 1e-5
    c.llm_layers, c.llm_hidden, c.llm_inter, c.llm_heads = m["layers"], m["hidden"], m["inter"], m["heads"]
    c.vocab, c.rms_eps, c.rope_theta = 32003, 1e-5, 10000.0
    c.proj_type, c.n_temporal = vn.PROJ_LINEAR, 100
    c.max_frames, c.max_batch, c.max_seq = 1, max_batch, S + N_NEW
    free0 = torch.cuda.mem_get_info()[0]
    eng = (binding or vn).Engine(c)
    own = llm is None
    if own:
        _, llm = bench.device_weights(model, "cuda")
    eng.load_llm(llm, weight_format=fmt)
    torch.cuda.synchronize()
    if own:
        del llm
        gc.collect()
        torch.cuda.empty_cache()
    return eng, free0 - torch.cuda.mem_get_info()[0]


def streamed_bytes(model, fmt):
    m = bench.MODELS[model]
    D, F, V, L = m["hidden"], m["inter"], 32003, m["layers"]
    mats = [(3 * D, D), (D, D), (2 * F, D), (D, F)] * L + [(V, D)]
    per = (lambda N, K: vn.tiled_elems(N, K) * 2) if fmt == "bf16" else (lambda N, K: vn.tiled_elems(N, K) + 4 * N)
    return sum(per(N, K) for N, K in mats)


def prompts(B, seed=1):
    ids = torch.cat([bench.synthetic_prompt_ids(seed=seed + b) for b in range(B)]).cuda()
    assert ids.shape[1] == S
    vf = (torch.randn(B, N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
          * 0.5).to(torch.bfloat16)
    vs = torch.full((B,), 64, dtype=torch.int32, device="cuda")
    return ids, vf, vs


def time_ms(fn, st):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(st):
        a.record(st)
        fn()
        b.record(st)
    b.synchronize()
    return a.elapsed_time(b)


def decode_arm(engines, B, rounds, st, model="7b", fmts=None):
    ids, vf, vs = prompts(B)
    firsts = {}
    with torch.cuda.stream(st):
        for k, e in engines.items():
            firsts[k] = e.prefill(ids, vf, vs)[2]
            e.decode_loop(firsts[k], S, N_NEW)                   # capture
    st.synchronize()
    times, toks = {k: [] for k in engines}, {}
    for _ in range(rounds):
        for k, e in engines.items():
            times[k].append(time_ms(lambda: toks.__setitem__(k, e.decode_loop(firsts[k], S, N_NEW)), st) / (N_NEW - 1))
    m = bench.MODELS[model]
    kv = 2 * m["layers"] * B * (S + N_NEW // 2) * m["hidden"] * 2       # K and V read per step, mean position
    out = {}
    for k in engines:
        ms = statistics.median(times[k])
        fmt = fmts[k] if fmts else k
        out[k] = dict(ms_per_step=round(ms, 3), gb_s=round((streamed_bytes(model, fmt) + kv) / ms / 1e6, 1),
                      spread_ms=[round(min(times[k]), 3), round(max(times[k]), 3)])
    if len(engines) > 1:
        ref = next(iter(engines))
        out["tokens_equal"] = all(torch.equal(firsts[k], firsts[ref]) and torch.equal(toks[k], toks[ref])
                                  for k in engines)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--skip-13b", action="store_true")
    ap.add_argument("--batches", default="1,4,16")
    ap.add_argument("--decode-only", action="store_true")
    ap.add_argument("--formats", default="bf16,fp8_e4m3")
    ap.add_argument("--compare-lib", default=None)
    ap.add_argument("--layers", type=int, default=None)
    args = ap.parse_args()
    if args.layers is not None:
        bench.MODELS["7b"] = dict(bench.MODELS["7b"], layers=args.layers)
    batches = [int(b) for b in args.batches.split(",")]
    formats = args.formats.split(",")
    name, power = card()
    print(f"[bench_fp8] {name}, power limit {power}")
    st = torch.cuda.Stream()
    res = {"card": name, "power_limit": power}

    _, llm = bench.device_weights("7b", "cuda")
    if args.compare_lib:
        other = other_binding(args.compare_lib)
        res["layers"] = bench.MODELS["7b"]["layers"]
        res["7b_decode_vs_other_lib"] = {}
        for fmt in formats:
            engines = {}
            engines["this"] = engine("7b", fmt, max_batch=max(batches + [16]), llm=llm)[0]
            engines["other"] = engine("7b", fmt, max_batch=max(batches + [16]), llm=llm, binding=other)[0]
            for B in batches:
                r = decode_arm(engines, B, args.rounds, st, fmts={"this": fmt, "other": fmt})
                r["speedup"] = round(r["other"]["ms_per_step"] / r["this"]["ms_per_step"], 3)
                res["7b_decode_vs_other_lib"][f"{fmt}_B{B}"] = r
                print(f"[bench_fp8] {fmt} B={B}: {r}", flush=True)
            for e in engines.values():
                e.close()
            del engines
            gc.collect()
            torch.cuda.empty_cache()
        print(json.dumps(res))
        return
    errs = []
    for k, v in llm.items():
        if k == "lm_head.weight" or (k.startswith("model.layers.") and k.endswith("_proj.weight")):
            d = R.dequantized(v)
            errs.append(((d.float() - v.float()).norm() ** 2).item() / (v.float().norm() ** 2).item())
    res["w_tilde_rel_err"] = round(statistics.mean(errs) ** 0.5, 4)
    engines, mems = {}, {}
    for fmt in formats:
        engines[fmt], mems[fmt] = engine("7b", fmt, max_batch=max(batches + [16]), llm=llm)
    del llm
    gc.collect()
    torch.cuda.empty_cache()
    res["7b_resident_gib"] = {k: round(v / 2 ** 30, 2) for k, v in mems.items()}
    res["7b_decode"] = {}
    for B in batches:
        r = decode_arm(engines, B, args.rounds, st)
        if len(engines) == 2:
            r["speedup"] = round(r["bf16"]["ms_per_step"] / r["fp8_e4m3"]["ms_per_step"], 3)
        res["7b_decode"][f"B{B}"] = r
        print(f"[bench_fp8] 7B decode B={B}: {r}")
    if args.decode_only:
        print(json.dumps(res))
        return
    eb, e8 = engines["bf16"], engines["fp8_e4m3"]

    # (b) one clip through the language model
    ids, vf, vs = prompts(1, seed=7)
    toks, t = {}, {k: [] for k in engines}
    for _ in range(args.rounds):
        for k, e in engines.items():
            t[k].append(time_ms(lambda: toks.__setitem__(k, e.generate(ids, vf, vs, N_NEW)), st))
    res["7b_llm_clips_per_s"] = {k: round(1000 / statistics.median(v), 3) for k, v in t.items()}
    # (c) fp8 against bf16 on W (random weights: report only)
    with torch.cuda.stream(st):
        lb = eb.prefill(ids, vf, vs, want_logits=True)[1]
        l8 = e8.prefill(ids, vf, vs, want_logits=True)[1]
    st.synchronize()
    res["fp8_vs_bf16_logits_rel_err"] = round(((l8 - lb).norm() / lb.norm()).item(), 4)
    res["fp8_vs_bf16_greedy_agreement"] = round((toks["bf16"] == toks["fp8_e4m3"]).float().mean().item(), 3)
    print(f"[bench_fp8] {res}")
    for e in engines.values():
        e.close()
    del engines, eb, e8
    gc.collect()
    torch.cuda.empty_cache()

    if not args.skip_13b:
        res["13b"] = {}
        for fmt in ("bf16", "fp8_e4m3"):
            e, mem = engine("13b", fmt, max_batch=4)
            res["13b"][f"resident_gib_{fmt}"] = round(mem / 2 ** 30, 2)
            if fmt == "fp8_e4m3":
                res["13b"]["fp8_decode_B4"] = decode_arm({fmt: e}, 4, args.rounds, st, model="13b")[fmt]
            e.close()
            del e
            gc.collect()
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Cost of scoring a sequence (vcl_llm_score: lm_head at every position + cross-entropy) next to the prefill.

    python tools/bench_score.py [--repeats 10] [--warmup 2] [--out DIR]

Vicuna-7B shapes with random-init bf16 weights (bench.device_weights, seed 0) and random video features; the
vision tower is not part of the measurement. Two workloads: 1 clip at S = 448 (bench.synthetic_prompt_ids), and 16
clips with prompt lengths spread over 400..448, left-padded to 448. Labels are -100 but on the last 26 tokens (the
answer part of the synthetic prompt). One engine (max_batch 16, max_seq 448) serves both, so its scoring tail runs
the lm_head GEMM over chunks of 2688 rows (one chunk for 1 clip, three for 16).
For each workload, alternated `--repeats` times after `--warmup` rounds, each timed with a host clock around the
call ended by a stream synchronise:
  prefill        vcl_llm_prefill(_padded), last-position logits (what forward returns without labels)
  score          vcl_llm_score with labels: per-token NLL and loss
  score_logits   the same, also writing the [B, S, 32003] bf16 logits (what forward(labels=...) returns)
  oracle         oracle/vcl_oracle.py on stock PyTorch, same GPU: llm_forward(all_logits=True) + F.cross_entropy
                 (unpadded: the oracle has no attention mask, so at 16 clips it runs 16 rows of 448)
The cross-entropy kernel alone (vcl_op_cross_entropy on a [rows, 32256] bf16 buffer, 448 and 7168 rows) is timed
with CUDA events over 50 launches; its bytes (logits read, labels read, NLL written) are computed from the shapes.
Prints one JSON line with the card name and power limit read in the same run.
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
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402
import vcl_native as vn  # noqa: E402
from bench_padded import card  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402

S_MAX, N_VID, N_ANSWER, V = 448, 356, 26, 32003


def make_engine(max_batch):
    m = bench.MODELS["7b"]
    c = vn.vcl_config()
    c.clip_layers, c.clip_hidden, c.clip_inter, c.clip_heads = 0, 1024, 4096, 16
    c.image_size, c.patch_size, c.clip_ln_eps = 224, 14, 1e-5
    c.llm_layers, c.llm_hidden, c.llm_inter, c.llm_heads = m["layers"], m["hidden"], m["inter"], m["heads"]
    c.vocab, c.rms_eps, c.rope_theta = V, 1e-5, 10000.0
    c.proj_type, c.n_temporal = vn.PROJ_LINEAR, 100
    c.max_frames, c.max_batch, c.max_seq = 1, max_batch, S_MAX
    eng = vn.Engine(c)
    clip, llm = bench.device_weights("7b", "cuda")
    del clip
    eng.load_llm(llm)
    return eng, llm


def workload(B, min_len=400):
    """B rows with lengths spread over min_len .. 448 (all 448 for one clip), left-padded with id 0"""
    lens = [S_MAX - round((S_MAX - min_len) * b / max(B - 1, 1)) for b in range(B)]
    ids = torch.zeros(B, S_MAX, dtype=torch.int64, device="cuda")
    full = torch.zeros(B, S_MAX, dtype=torch.int64, device="cuda")       # the unpadded rows (the oracle's input)
    for b, n in enumerate(lens):
        r = bench.synthetic_prompt_ids(seed=1 + b, n_pre=63 - (S_MAX - n)).cuda()
        ids[b, S_MAX - n:] = r[0]
        full[b] = bench.synthetic_prompt_ids(seed=1 + b).cuda()[0]
    pads = [S_MAX - n for n in lens]
    vs = torch.full((B,), 64, dtype=torch.int32, device="cuda")          # <vid_start> column of every padded row
    lab = torch.full_like(ids, -100)
    lab[:, -N_ANSWER:] = ids[:, -N_ANSWER:]
    lab_full = torch.full_like(full, -100)
    lab_full[:, -N_ANSWER:] = full[:, -N_ANSWER:]
    return ids, (pads if any(pads) else None), vs, lab, full, lab_full


def ce_kernel(rows, iters=50):
    x = (torch.randn(rows, 32256, device="cuda") * 3).to(torch.bfloat16)
    lab = torch.randint(0, V, (rows,), device="cuda")
    for _ in range(3):
        vn.op_cross_entropy(x, lab, V=V, want_loss=False)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        vn.op_cross_entropy(x, lab, V=V, want_loss=False)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    nbytes = rows * V * 2 + rows * 8 + rows * 4
    return {"rows": rows, "us": round(us, 1), "bytes": nbytes, "GB_per_s": round(nbytes / us / 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON line to DIR/bench_score.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_score.py needs an H100 (no CPU measurement)")
    name, power = card()
    eng, llm = make_engine(16)
    cfg = O.LlmCfg()
    st = torch.cuda.Stream()
    res = {"what": "Vicuna-7B shapes, random bf16 weights, video features given, labels on the last 26 tokens",
           "card": name, "power_limit": power, "repeats": a.repeats, "warmup": a.warmup}

    def timed(fn):
        st.synchronize()
        t0 = time.perf_counter()
        with torch.cuda.stream(st):
            out = fn()
        st.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    for B in (1, 16):
        ids, pads, vs, lab, full, lab_full = workload(B)
        vf = (torch.randn(B, N_VID, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))
              * 0.5).to(torch.bfloat16)
        arms = {
            "prefill": lambda: eng.prefill(ids, vf, vs, want_logits=True, want_token=False, n_pad=pads),
            "score": lambda: eng.score(ids, vf, vs, labels=lab, n_pad=pads),
            "score_logits": lambda: eng.score(ids, vf, vs, labels=lab, n_pad=pads, want_logits=True),
        }

        def oracle():
            lg, _, _ = O.llm_forward(llm, cfg, full, vf, all_logits=True)
            return F.cross_entropy(lg[:, :-1].reshape(-1, V), lab_full[:, 1:].reshape(-1))

        with torch.no_grad():
            times = {k: [] for k in list(arms) + ["oracle"]}
            for i in range(a.warmup + a.repeats):
                for k, fn in list(arms.items()) + [("oracle", oracle)]:
                    t, out = timed(fn)
                    if i >= a.warmup:
                        times[k].append(t)
                    if k == "score":
                        loss = out[2]
                    if k == "oracle":
                        o_loss = out
        med = {k: statistics.median(v) for k, v in times.items()}
        res[f"clips_{B}"] = {
            "pads": pads or [0] * B,
            **{f"{k}_ms": {"min": round(min(v), 2), "median": round(med[k], 2)} for k, v in times.items()},
            "score_minus_prefill_ms": round(med["score"] - med["prefill"], 2),
            "score_logits_minus_prefill_ms": round(med["score_logits"] - med["prefill"], 2),
            "oracle_over_score_logits": round(med["oracle"] / med["score_logits"], 2),
            "loss": round(loss.item(), 5),
            "oracle_loss_unpadded": round(o_loss.float().item(), 5),
        }
        del vf
        torch.cuda.empty_cache()
    res["ce_kernel"] = [ce_kernel(448), ce_kernel(7168)]
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_score.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

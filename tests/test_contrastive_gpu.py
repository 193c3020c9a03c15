"""GPU tests of contrastive search: vcl_op_contrastive_rank against the float64 rule (_contrastive_ref.py) on random
and adversarial inputs, the engine's steps against the oracle's float64 restatement with the near-tie rule (teacher
forced with the device's picks), the prompt's k clips holding the same cache columns after every call, a left-padded
batch against its rows run alone, chunked graphs against eager steps, generate() with EOS and stopping criteria, and a
greedy call after a contrastive one against a fresh engine."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "video-llava_b200"))

import vcl_native as vn  # noqa: E402
import _contrastive_ref as CR  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import make_engine, to_dev, vid_start_of  # noqa: E402
from test_inflight_gpu import text_prompt  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)


@pytest.fixture(autouse=True)
def _release():
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


def _rank_inputs(B, k, D, n_ctx, kind, seed):
    g = torch.Generator().manual_seed(seed)
    ctx = torch.randn(B, n_ctx + 1, D, generator=g)
    hid = torch.randn(B * k, D, generator=g)
    p = torch.rand(B * k, generator=g) * 0.2
    pads = [(5 * b) % max(1, n_ctx // 2) for b in range(B)]
    if kind == "parallel":              # candidates nearly parallel to a context row: cosines near 1, close together
        for b in range(B):
            for j in range(k):
                hid[b * k + j] = ctx[b, n_ctx - 1 - j % 3] * (1 + 0.01 * j) + 1e-3 * torch.randn(D, generator=g)
    elif kind == "duplicate":           # two candidates with the same row and probability: the lower j wins the tie
        for b in range(B):
            hid[b * k + 1] = hid[b * k]
            p[b * k + 1] = p[b * k]
            p[b * k] = p[b * k + 1] = 0.9
    elif kind == "all_pad":             # one real context row per prompt
        pads = [n_ctx - 1] * B
    tok = torch.randint(0, 32000, (B * k,), generator=g, dtype=torch.int32)
    return ctx.to(torch.bfloat16), hid.to(torch.bfloat16), p.float(), tok, pads


@torch.no_grad()
@pytest.mark.parametrize("D", [4096, 5120])
@pytest.mark.parametrize("B,k", [(1, 2), (2, 4), (3, 6), (1, 8), (2, 16), (1, 64)])
@pytest.mark.parametrize("kind", ["random", "parallel", "duplicate", "all_pad"])
def test_rank_matches_fp64_rule(D, B, k, kind):
    n_ctx, alpha = 300, 0.6
    ctx, hid, p, tok, pads = _rank_inputs(B, k, D, n_ctx, kind, seed=D + 7 * B + k)
    c_dev = ctx.to(DEV)
    rec = vn.op_contrastive_rank(c_dev, pads, n_ctx, hid.to(DEV), p.to(DEV), tok.to(DEV), alpha)
    r = {n: v.cpu() for n, v in vn.cs_records(rec, k).items()}
    c_dev = c_dev.cpu()
    for b in range(B):
        rows = ctx[b, pads[b]:n_ctx].double().numpy()
        g = hid[b * k:(b + 1) * k].double().numpy()
        s, score, j = CR.rank(rows, g, p[b * k:(b + 1) * k].double().numpy(), alpha)
        assert np.abs(r["cos"][b].double().numpy() - s).max() <= 2e-6, (b, r["cos"][b], s)
        assert np.abs(r["score"][b].double().numpy() - score).max() <= 2e-6
        assert r["cand"][b].tolist() == tok[b * k:(b + 1) * k].tolist()
        pick = int(r["pick"][b])
        if CR.decided(score, j, lambda x, y: 1e-5):
            assert pick == j, (b, pick, j, score)
        else:
            assert score[j] - score[pick] <= 1e-5
        if kind == "duplicate":
            assert pick != 1 or float(r["score"][b, 0]) < float(r["score"][b, 1])
        assert int(r["token"][b]) == int(tok[b * k + pick])
        # the chosen row is appended to the context, bit for bit
        assert torch.equal(c_dev[b, n_ctx].view(torch.int16), hid[b * k + pick].view(torch.int16))


# ------------------------------------------------------------------------------------------
def _engine(max_batch, cfg=SMALL, sd=None, max_seq=160):
    eng = make_engine(llm=cfg, max_batch=max_batch, max_seq=max_seq)
    eng.load_llm(sd if sd is not None else to_dev(O.random_llm_state(cfg, seed=21)))
    return eng


def _prompts(B, padded, S=24):
    ids = torch.stack([text_prompt(700 + b, S) for b in range(B)]).to(DEV)
    pads = [(3 * b) % 7 for b in range(B)] if padded else None
    return ids, pads


def _run(eng, ids, pads, k, alpha, chunks, cfg=SMALL):
    vs = vid_start_of(ids, cfg)
    tok, rec = eng.contrastive_start(ids, None, vs, k, alpha, 1 + sum(chunks), n_pad=pads)
    toks, recs = [tok], [rec]
    for c in chunks:
        t, r = eng.contrastive_decode(c)
        toks.append(t)
        recs.append(r)
    return torch.cat(toks).cpu(), torch.cat(recs).cpu()


@torch.no_grad()
@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("k,alpha", [(4, 0.6), (2, 1.0), (8, 0.3)])
def test_engine_matches_oracle_restatement(wide, k, alpha):
    """each step's candidates and pick against the float64 rule on the bf16 oracle's hidden rows and logits, teacher
    forced with the device's tokens: a candidate place must match wherever the oracle's p separates it from its
    neighbours, and the float64 pick among the device's candidates wherever its score is apart from every other by
    the stated margin"""
    cfg = O.LlmCfg(hidden=4096, inter=11008, heads=32, layers=2) if wide else SMALL
    sd = to_dev(O.random_llm_state(cfg, seed=5))
    eng = _engine(k, cfg, sd)
    ids, _ = _prompts(1, False)
    n = 16
    tok, rec = _run(eng, ids, None, k, alpha, [n - 1], cfg)
    r = vn.cs_records(rec[:, 0], k)
    step, ctx0, z0 = CR.oracle_step_fn(sd, cfg, ids, None)
    ctx, z, chosen, worst = ctx0, z0, [], 0.0
    places = ok_places = picks = ok_picks = 0
    for t in range(n):
        cand, p = CR.candidates(z, k)
        lz = np.log(p)                   # a place counts where log p is 0.25 apart on both sides (two bf16 ulps of a
        #                                  logit below 16, twice)
        for q in range(k):
            if (q == 0 or lz[q - 1] - lz[q] > 0.25) and (q + 1 == k or lz[q] - lz[q + 1] > 0.25):
                places += 1
                ok_places += int(r["cand"][t, q]) == int(cand[q])
        # the rank on the device's candidates, with the oracle's rows and probabilities
        dc = r["cand"][t].numpy()
        g, zs = step(chosen, dc)
        pz = CR.probs(z)[dc]
        s, score, j = CR.rank(ctx, g, pz, alpha)
        e_cos = np.abs(r["cos"][t].double().numpy() - s).max()
        e_p = np.abs(r["p"][t].double().numpy() - pz).max()
        assert e_cos <= 0.02 and e_p <= 0.05 * pz.max(), (t, r["cos"][t], s, r["p"][t], pz)
        worst = max(worst, e_cos)
        # decided: the gap exceeds twice what the measured input differences can move a score
        margin = lambda a, b: 2 * (alpha * e_cos + (1 - alpha) * e_p) + 1e-6   # noqa: E731
        if CR.decided(score, j, margin):
            picks += 1
            ok_picks += int(r["pick"][t]) == j
        jd = int(r["pick"][t])                               # teacher forced with the device's pick
        chosen.append(int(dc[jd]))
        ctx = np.concatenate([ctx, g[jd][None]], axis=0)
        z = zs[jd]
    print(f"[contrastive] wide {wide} k {k} a {alpha}: {ok_places}/{places} decided candidate places, "
          f"{ok_picks}/{picks} decided picks of {n} steps, cosines within {worst:.2e}")
    assert ok_places == places and ok_picks == picks
    assert places >= 3 and picks >= n // 2


@torch.no_grad()
@pytest.mark.parametrize("B,k,padded", [(1, 4, False), (2, 3, True), (3, 8, True), (9, 8, False)])
def test_clips_hold_the_same_columns(B, k, padded):
    eng = _engine(B * k, max_seq=96)
    ids, pads = _prompts(B, padded)
    S, n = ids.shape[1], 20
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        _run(eng, ids, pads, k, 0.6, [7, 12])
    st.synchronize()
    for layer in range(SMALL.layers):
        kc, vc = eng.kv_cache(layer)
        for b in range(B):
            clips = [b] + [B + b * (k - 1) + j - 1 for j in range(1, k)]
            for c in clips[1:]:
                for x in (kc, vc):
                    assert torch.equal(x[c, :, :S + n].view(torch.int16), x[b, :, :S + n].view(torch.int16)), \
                        (layer, b, c)


@torch.no_grad()
def test_padded_batch_rows_equal_rows_alone():
    k = 4
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    eng = _engine(3 * k, sd=sd)
    lens = [24, 19, 13]
    rows = [text_prompt(900 + b, L).to(DEV) for b, L in enumerate(lens)]
    S = max(lens)
    ids = torch.stack([torch.cat([torch.zeros(S - len(r), dtype=r.dtype, device=DEV), r]) for r in rows])
    pads = [S - L for L in lens]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        tb, rb = _run(eng, ids, pads, k, 0.6, [15])
        alone = [_run(eng, r[None], None, k, 0.6, [15]) for r in rows]
    st.synchronize()
    for b in range(3):
        assert torch.equal(tb[:, b], alone[b][0][:, 0]), (b, tb[:, b], alone[b][0][:, 0])


@torch.no_grad()
def test_graph_chunks_and_eager_steps_agree():
    B, k = 2, 4
    eng = _engine(B * k)
    ids, pads = _prompts(B, True)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        g1 = _run(eng, ids, pads, k, 0.6, [29])
        g2 = _run(eng, ids, pads, k, 0.6, [5, 8, 16])
    st.synchronize()
    e = _run(eng, ids, pads, k, 0.6, [1] * 29)     # the legacy default stream cannot be captured: eager steps
    torch.cuda.synchronize()
    for g in (g1, g2):
        assert torch.equal(g[0], e[0]) and torch.equal(g[1].view(torch.int32), e[1].view(torch.int32))


def _model(eng, max_batch):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=SMALL.hidden, intermediate_size=SMALL.inter, num_hidden_layers=SMALL.layers,
                             num_attention_heads=SMALL.heads, vocab_size=SMALL.vocab, eos_token_id=2)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=max_batch, max_seq=160)
    m._engine, m._llm_loaded = eng, True
    return m


@torch.no_grad()
def test_generate_eos_stops_and_greedy_after_is_fresh():
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    ids, _ = _prompts(2, False)
    eng = _engine(8, sd=sd)
    tok, _ = _run(eng, ids, None, 4, 0.6, [39])
    m = _model(eng, 8)
    eos = int(tok[5, 0])                           # row 0's sixth token
    out = m.generate(ids, max_new_tokens=40, eos_token_id=eos, pad_token_id=0, penalty_alpha=0.6, top_k=4)
    S = ids.shape[1]
    new = out[:, S:].cpu()
    ref = tok.T.clone().to(torch.int64)
    for b in range(2):
        hit = (ref[b] == eos).nonzero()
        if len(hit):
            ref[b, int(hit[0]) + 1:] = 0
    stop = max(int((ref[b] == eos).nonzero()[0]) if (ref[b] == eos).any() else 39 for b in range(2)) + 1
    assert torch.equal(new, ref[:, :stop]), (new, ref)

    class Stop:                                     # stop after the 3rd new token
        def __call__(self, seq, scores):
            return seq.shape[1] >= S + 3
    out2 = m.generate(ids, max_new_tokens=40, eos_token_id=None, stopping_criteria=[Stop()], penalty_alpha=0.6,
                      top_k=4)
    assert torch.equal(out2[:, S:].cpu(), tok.T[:, :3].to(torch.int64))
    with pytest.raises(ValueError, match="contrastive"):
        m.generate_continue(ids[:, :3])

    fresh = _engine(8, sd=sd)
    vs = vid_start_of(ids, SMALL)
    st = torch.cuda.Stream()

    def counted(e):
        st.synchronize()
        n0 = vn.launch_count()
        out = e.generate(ids, None, vs, 9)
        st.synchronize()
        return out, vn.launch_count() - n0

    with torch.cuda.stream(st):
        g0, n0 = counted(eng)
        g1, n1 = counted(fresh)
    assert torch.equal(g0, g1) and n0 == n1


def test_rejections():
    eng = _engine(4)
    ids, _ = _prompts(1, False)
    vs = vid_start_of(ids, SMALL)
    n0 = vn.launch_count()
    for k, a, n, why in ((1, 0.6, 8, "top_k"), (65, 0.6, 8, "top_k"), (8, 0.6, 8, "max_batch"),
                         (2, 0.0, 8, "penalty_alpha"), (2, 1.5, 8, "penalty_alpha"), (2, 0.6, 137, "max_seq")):
        with pytest.raises(vn.VclError, match=why):
            eng.contrastive_start(ids, None, vs, k, a, n)
    eng._cs_shape = (1, 2)
    with pytest.raises(vn.VclError, match="no contrastive search"):
        eng.contrastive_decode(1)
    assert vn.launch_count() == n0

"""score_candidates on the H100: the label log-prob kernel (vcl_op_label_logprobs) against float64 and against the
sampler's own log-probs, the contiguous packed flash instance (vcl_op_attention_appended) bit for bit against the
continued prefill, and the whole call: packing invariance, cache isolation, the bf16 oracle at 7B and 13B width,
greedy answers, fp8 weights and the engine state afterwards."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _fp8_ref as F8  # noqa: E402
import _logprob_ref as R  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import to_dev  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
W7B = O.LlmCfg(hidden=4096, inter=11008, heads=32, layers=2)
W13B = O.LlmCfg(hidden=5120, inter=13824, heads=40, layers=1)


# ------------------------------------------------------------------------------------------------
# the kernel
def _rows(V, seed):
    """bf16 rows: random, exact ties at the top (first, middle, last index), a NaN row, an all -inf row, NaNs and -inf
    inside a row, a one-hot row"""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(24, V, generator=g) * 3).bfloat16()
    top = x.float().max().item() + 1
    x[1, [7, V // 2, V - 1]] = top                         # ties: the label at each of them below
    x[2, [0, 1]] = top
    x[3] = float("nan")
    x[4] = float("-inf")
    x[5, ::3] = float("nan")
    x[6, ::2] = float("-inf")
    x[7] = -30.0
    x[7, V // 3] = 50.0
    x[8, V - 1] = top                                     # the maximum at the last index
    return x


def _labels(x, seed):
    V = x.shape[1]
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, V, (x.shape[0],), generator=g)
    xf = x.float().nan_to_num(nan=-float("inf"))
    am = xf.argmax(-1)                                    # torch: the first maximal index
    for r in range(0, x.shape[0], 2):
        lab[r] = am[r]
    lab[1], lab[2], lab[8] = V // 2, 0, V - 1
    lab[9] = V - 1
    return lab


@torch.no_grad()
@pytest.mark.parametrize("V", [32003, 1000])
def test_label_logprobs_kernel(V):
    x = _rows(V, V)
    lab = _labels(x, V + 1)
    # ties: label 1 is the middle of three tied maxima (not greedy); row 2's label 0 is the first (greedy)
    lp, greedy = vn.op_label_logprobs(x.to(DEV), lab.to(DEV))
    lp, greedy = lp.cpu().numpy(), greedy.cpu().numpy()
    xf = x.float().numpy()
    for r in range(x.shape[0]):
        want, _, _ = R.logprobs(xf[r], 0.0, 0, 0, int(lab[r]))
        if np.isnan(xf[r, int(lab[r])]):
            want = float("nan")                               # a NaN logit at the label: (NaN - m) - log W
        assert R.close(lp[r], want), (r, lp[r], want)
        row = np.where(np.isnan(xf[r]), -np.inf, xf[r])
        finite = np.isfinite(row.max())
        assert bool(greedy[r]) == (finite and int(np.argmax(row)) == int(lab[r])), (r, greedy[r])
    assert greedy[2] and not greedy[1] and greedy[8] and np.isnan(lp[3]) and np.isnan(lp[4]) and not greedy[3]
    # the sampler's chosen-token value at T = 0 is the arg-max's: bit for bit wherever the label is the arg-max
    B = x.shape[0]
    tok, _, slp = vn.op_sample_logprobs(x.float().to(DEV), [0.0] * B, [0] * B, [0] * B, [0] * B, [0] * B)
    tok, slp = tok.cpu(), slp[:, 0].cpu()
    n = 0
    for r in range(B):
        if int(tok[r]) == int(lab[r]) and greedy[r]:
            assert np.float32(slp[r]).tobytes() == np.float32(lp[r]).tobytes(), r
            n += 1
    assert n >= B // 2 - 3
    # a padded row pitch and labels outside the vocabulary
    xp = torch.zeros(3, V + 13, dtype=torch.bfloat16)
    xp[:, :V] = x[:3]
    lp2, g2 = vn.op_label_logprobs(xp.to(DEV), torch.tensor([int(lab[0]), -1, V]).to(DEV), V=V)
    assert lp2[0].item() == lp[0] and torch.isnan(lp2[1:]).all() and not g2[1:].any()


# ------------------------------------------------------------------------------------------------
# the contiguous packed flash instance
APPENDED = [(3, 500, 37), (0, 511, 1), (5, 600, 100), (1, 1000, 24), (6, 1500, 300), (2, 1900, 148), (4, 100, 50)]


@torch.no_grad()
def test_appended_attention_matches_the_continued_prefill():
    """every sequence bit for bit against vcl_op_attention_cached at the same start, in a clip of its own; columns
    past each sequence's end and the unowned slot 7 are NaN"""
    H, s_max, n_slots = 2, 2048, 8
    g = torch.Generator(device=DEV).manual_seed(3)
    k = torch.randn(n_slots, H, s_max, 128, device=DEV, generator=g).bfloat16()
    v = torch.randn(n_slots, H, s_max, 128, device=DEV, generator=g).bfloat16()
    for s, st, n in APPENDED:
        k[s, :, st + n:] = float("nan")
        v[s, :, st + n:] = float("nan")
    k[7] = float("nan")
    v[7] = float("nan")
    M = sum(n for _, _, n in APPENDED)
    q = torch.randn(M, 3 * H * 128, device=DEV, generator=g).bfloat16()
    slots, starts, lens = zip(*APPENDED)
    n0 = vn.launch_count()
    o = vn.op_attention_appended(q, k, v, slots, starts, lens)
    torch.cuda.synchronize()
    assert vn.launch_count() - n0 == 2                      # one wgmma and one flash launch
    assert torch.isfinite(o.float()).all()
    off = 0
    for s, st, n in APPENDED:
        alone = vn.op_attention_cached(q[off:off + n], k[s:s + 1].contiguous(), v[s:s + 1].contiguous(), st)
        assert torch.equal(alone, o[off:off + n]), (s, st, n)
        off += n


# ------------------------------------------------------------------------------------------------
# the whole call
def _model(cfg, max_slots=4, max_seq=800, fmt="bf16"):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    c = VideoChatGPTConfig(hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers,
                           num_attention_heads=cfg.heads, vocab_size=cfg.vocab, use_mm_proj=True, mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    m = VideoChatGPTLlamaForCausalLM(c, clip_config=clip, max_batch=max_slots, max_seq=max_seq, max_slots=max_slots,
                                     llm_weight_format=fmt)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    return m


def _questions(cfg, n_post, seed, n_opts=5):
    """prompts of 63 + 358 + n_post tokens with video, and n_opts seeded options of 1 .. 32 tokens each"""
    out = []
    for i, post in enumerate(n_post):
        ids = O.make_prompt_ids(cfg, 356, seed=seed + i, n_post=post)[0]
        g = torch.Generator().manual_seed(seed * 7 + i)
        lens = [1] + torch.randint(2, 33, (n_opts - 1,), generator=g).tolist()
        opts = [torch.randint(3, 31990, (L,), generator=g) for L in lens]
        out.append((ids, opts, video_feats(1, seed + i)[0]))
    return out


def _call(m, qs):
    return m.score_candidates([q[0] for q in qs], [q[1] for q in qs],
                              video_spatio_temporal_features=[q[2] for q in qs])


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous().view(torch.int64)


def _same_option(a, b, i, j, what):
    assert torch.equal(_bits(a["token_logprobs"][i]), _bits(b["token_logprobs"][j])), what
    assert bool(a["greedy"][i]) == bool(b["greedy"][j]), what
    assert a["logprob"][i].view(torch.int64) == b["logprob"][j].view(torch.int64), what


@pytest.fixture(scope="module")
def small():
    sd = to_dev(O.random_llm_state(SMALL, seed=7))
    ms = {}
    for n in (4, 2):
        m = _model(SMALL, max_slots=n)
        m.load_state_dict(sd)
        m._ensure_engine(need_llm=True)
        ms[n] = m
    yield ms
    for m in ms.values():
        m._engine.close()


@torch.no_grad()
def test_packing_invariance(small):
    """prompts of <= 512 and > 512 tokens; each option equals a one-option call of it, whatever its slot, neighbours,
    prompt order or round split"""
    qs = _questions(SMALL, [26, 250, 60], seed=31)           # 447, 671 and 481 tokens
    full = _call(small[4], qs)
    rev = _call(small[4], qs[::-1])
    split = _call(small[2], qs)
    for b, (ids, opts, f) in enumerate(qs):
        for j, c in enumerate(opts):
            alone = small[4].score_candidates([ids], [[c]], video_spatio_temporal_features=[f])[0]
            _same_option(full[b], alone, j, 0, f"prompt {b} option {j}")
            _same_option(rev[len(qs) - 1 - b], alone, j, 0, f"reversed: prompt {b} option {j}")
            _same_option(split[b], alone, j, 0, f"max_slots 2: prompt {b} option {j}")
            assert torch.isfinite(full[b]["token_logprobs"][j]).all()


@torch.no_grad()
def test_cache_isolation(small):
    """a call writes only the slots it uses; the prompt slot's columns 0 .. S - 2 keep the prefill's bits across the
    rounds that fork from it (max_slots 2: five options over four rounds)"""
    m = small[2]
    eng = m._engine
    (ids, opts, f), = _questions(SMALL, [40], seed=77)
    S = ids.numel()
    eng.slots_prefill([0], [ids], [f], [m._video_spans(ids[None], eng.NV)[0]])
    want = [eng.kv_cache(layer) for layer in range(SMALL.layers)]
    m.score_candidates([ids], [opts], video_spatio_temporal_features=[f])
    for layer in range(SMALL.layers):
        k, v = eng.kv_cache(layer)
        for got, ref in ((k, want[layer][0]), (v, want[layer][1])):
            assert torch.equal(got[0, :, :S - 1].view(torch.int16), ref[0, :, :S - 1].view(torch.int16))
            assert torch.equal(got[1, :, :S - 1].view(torch.int16), ref[0, :, :S - 1].view(torch.int16))
    # a one-prompt call on the 4-slot engine: 2 options use slots 0 and 1; slots 2 and 3 keep a NaN sentinel
    m4 = small[4]
    e4 = m4._engine
    nan = torch.full(e4._cache_shape(), 0x7FC1, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    for layer in range(SMALL.layers):
        e4.set_kv_cache(layer, nan, nan)
    m4.score_candidates([ids], [opts[:2]], video_spatio_temporal_features=[f])
    for layer in range(SMALL.layers):
        k, v = e4.kv_cache(layer)
        for t in (k, v):
            assert (t[2:].view(torch.int16) == 0x7FC1).all()
            assert (t[:2, :, S + 32:].view(torch.int16) == 0x7FC1).all()
            assert torch.isfinite(t[:2, :, :S - 1].float()).all()


def _margin_ulps(logits):
    top = torch.topk(logits.float(), 2, dim=-1).values
    return (top[..., 0] - top[..., 1]) / (top[..., 0].abs().clamp_min(2 ** -6) * 2 ** -7)


@torch.no_grad()
@pytest.mark.parametrize("cfg", [W7B, W13B], ids=["7b", "13b"])
def test_against_the_bf16_oracle(cfg):
    sd = to_dev(O.random_llm_state(cfg, seed=5))
    m = _model(cfg, max_slots=4, max_seq=480)
    m.load_state_dict(sd)
    qs = _questions(cfg, [26, 10, 5], seed=91, n_opts=4)
    for ids, opts, f in qs:   # one more option: the oracle's own top-1 token after the prompt
        lg, _, _ = O.llm_forward(sd, cfg, ids[None].to(DEV), f[None].to(DEV).bfloat16(), all_logits=True)
        opts.append(lg[0, -1].float().argmax().reshape(1).cpu())
    out = _call(m, qs)
    n_pos = 0
    for b, (ids, opts, f) in enumerate(qs):
        S = ids.numel()
        for j, c in enumerate(opts):
            seq = torch.cat([ids, c])[None].to(DEV)
            logits, _, _ = O.llm_forward(sd, cfg, seq, f[None].to(DEV).bfloat16(), all_logits=True)
            rows = logits[0, S - 1:S - 1 + c.numel()].float()
            want = torch.log_softmax(rows, -1)[torch.arange(c.numel()), c.to(DEV)]
            got = out[b]["token_logprobs"][j].to(DEV)
            err = (got - want).abs().max().item()
            print(f"[candidates] width {cfg.hidden}: prompt {b} option {j} ({c.numel()} tokens): max |lp - oracle| "
                  f"{err:.3e}")
            assert err < 3e-2 * max(1.0, want.abs().max().item()), (b, j, err)
            decided = _margin_ulps(rows) >= 3
            o_greedy = rows.argmax(-1) == c.to(DEV)
            if decided.all():
                assert bool(out[b]["greedy"][j]) == bool(o_greedy.all()), (b, j)
                n_pos += bool(o_greedy.all())
            elif not (o_greedy | ~decided).all():
                assert not out[b]["greedy"][j], (b, j)
    print(f"[candidates] width {cfg.hidden}: {n_pos} of {len(qs)} top-1 options decided by the margin rule and greedy")
    assert n_pos >= 1                                      # the positive case ran
    m._engine.close()


@torch.no_grad()
def test_greedy_answer_is_greedy(small):
    """each token of generate's greedy answer, scored as a one-token option after the prompt and the answer's earlier
    tokens, is greedy wherever the engine's own logits decide it (top-1 / top-2 margin >= 3 bf16 ulps), and the next
    token id is not; at least one step must be decided"""
    m = small[4]
    (ids, _, f), = _questions(SMALL, [26], seed=5)
    n = 8
    gen = m.generate(ids[None].to(DEV), f[None].to(DEV), max_new_tokens=n, eos_token_id=None)
    ans = gen[0, ids.numel():].cpu()
    prompts = [torch.cat([ids, ans[:t]]) for t in range(n)]
    cands = [[ans[t:t + 1], (ans[t:t + 1] + 1) % 31990] for t in range(n)]
    out = m.score_candidates(prompts, cands, video_spatio_temporal_features=[f] * n)
    lg = m.forward(torch.cat([ids, ans])[None].to(DEV), video_spatio_temporal_features=f[None].to(DEV),
                   logits_to_keep=0).logits[0, ids.numel() - 1:-1]
    decided = (_margin_ulps(lg) >= 3).tolist()
    print(f"[candidates] greedy answer: {sum(decided)} of {n} steps decided by the margin rule")
    for t in range(n):
        if decided[t]:
            assert out[t]["greedy"].tolist() == [True, False], t
    assert sum(decided) >= 1


@torch.no_grad()
def test_one_token_prompt(small):
    """a BOS-only prompt (lm-eval's empty context): its options start at column 0 of their slots, next to a longer
    prompt in the same round; each equals a one-option call and the log-softmax of the engine's own logits"""
    m = small[4]
    (ids, opts, f), = _questions(SMALL, [26], seed=17, n_opts=2)
    bos = torch.tensor([1])
    g = torch.Generator().manual_seed(2)
    bos_opts = [torch.randint(3, 31990, (L,), generator=g) for L in (1, 9)]
    out = m.score_candidates([bos, ids], [bos_opts, opts], video_spatio_temporal_features=[None, f])
    for j, c in enumerate(bos_opts):
        alone = m.score_candidates([bos], [[c]])[0]
        _same_option(out[0], alone, j, 0, f"one-token prompt, option {j}")
        lg = m.forward(torch.cat([bos, c])[None].to(DEV), logits_to_keep=0).logits[0, :c.numel()].float()
        want = torch.log_softmax(lg, -1)[torch.arange(c.numel()), c.to(DEV)].cpu()
        torch.testing.assert_close(out[0]["token_logprobs"][j], want, rtol=1e-5, atol=1e-5)
    for j, c in enumerate(opts):
        alone = m.score_candidates([ids], [[c]], video_spatio_temporal_features=[f])[0]
        _same_option(out[1], alone, j, 0, f"video prompt next to the one-token prompt, option {j}")


@torch.no_grad()
def test_fp8_equals_bf16_on_dequantized_weights():
    sd = to_dev(O.random_llm_state(W7B, seed=41))
    m8, mb = _model(W7B, 4, 480, "fp8_e4m3"), _model(W7B, 4, 480)
    m8.load_state_dict(sd)
    mb.load_state_dict(F8.dequantize_state(sd))
    qs = _questions(W7B, [26, 12], seed=13)
    a, b = _call(m8, qs), _call(mb, qs)
    for i in range(len(qs)):
        for j in range(len(qs[i][1])):
            _same_option(a[i], b[i], j, j, f"fp8 vs bf16 on W~: prompt {i} option {j}")
    m8._engine.close()
    mb._engine.close()


@torch.no_grad()
def test_generate_after_scoring(small):
    """a generate after score_candidates returns a fresh engine's tokens with a fresh engine's launch count"""
    (ids, opts, f), = _questions(SMALL, [26], seed=3)
    sd = to_dev(O.random_llm_state(SMALL, seed=7))
    fresh = _model(SMALL, max_slots=4)
    fresh.load_state_dict(sd)
    x, fx = ids[None].to(DEV), f[None].to(DEV)
    fresh.generate(x, fx, max_new_tokens=4, eos_token_id=None)       # warm the graph cache of both engines alike
    m = small[4]
    m.generate(x, fx, max_new_tokens=4, eos_token_id=None)
    n0 = vn.launch_count()
    want = fresh.generate(x, fx, max_new_tokens=12, eos_token_id=None)
    n_want = vn.launch_count() - n0
    m.score_candidates([ids], [opts], video_spatio_temporal_features=[f])
    with pytest.raises(ValueError, match="no previous generate"):
        m.generate_continue(torch.tensor([[5, 6]], device=DEV))
    n0 = vn.launch_count()
    got = m.generate(x, fx, max_new_tokens=12, eos_token_id=None)
    assert vn.launch_count() - n0 == n_want
    assert torch.equal(got.cpu(), want.cpu())
    fresh._engine.close()

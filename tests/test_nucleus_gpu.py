"""Top-p and the repetition penalty on the GPU (sampling.cu's 32-bit path, vcl_llm_set_sampling_ex, token sets).

Bars:
- the kernel against the float64 rules of _nucleus_ref.py: a sampled token is always in the fp64 final kept set and
  is the fp64 choice wherever u * W' lies at least 1e-5 W' from its interval's edges; a greedy penalized row is
  torch's arg-max of the penalized fp32 logits; a row with p = 1, r = 1 equals vcl_op_sample(_logprobs) bit for bit;
  the picked token joins the row's token set; on rows whose top-p boundary is decided, the log-prob alternatives
  are exactly the fp64 kept set's largest tokens;
- a chi-square test of one row with top-p and a penalty against its exact probabilities;
- token sets read back after generate (plain and left-padded), generate_continue, a session's turns and a chunked
  prompt equal the sequence's ids; a chunked prompt's tokens equal a one-shot prefill's;
- end to end, at every step that a 3-ulp move of the logits cannot change: the token of generate, generate_continue
  and generate_requests (top_p 0.9, penalty 1.3, T 0.7) is the one HF's own processors on the bf16 oracle's logits
  give for the same u, on bf16 and fp8 engines;
- greedy generate with a penalty, teacher-forced on the engine's own scored logits, picks the arg-max of the
  penalized logits at every step whose top-2 gap exceeds 3 bf16 ulps;
- bit-identical reproducibility across slots, neighbours and admission mode; a default call after a penalized one
  equals a fresh engine's, with the same launch count; the C ABI rejections.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _nucleus_ref as N  # noqa: E402
import _sampling_ref as R  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import to_dev  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402
from test_inflight_gpu import _model, _requests  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)


def _rows(B, V, seed, scale):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, V, generator=g) * scale[:, None]).bfloat16().float()


def _bits(sets, V):
    """token-set lists -> [B, words] int32 bitmaps"""
    words = vn.token_set_words(V)
    out = np.zeros((len(sets), words), dtype=np.uint32)
    for b, s in enumerate(sets):
        for t in s:
            out[b, t >> 5] |= np.uint32(1 << (t & 31))
    return torch.from_numpy(out.view(np.int32)).to(DEV)


def _unbits(bits, V):
    b = bits.cpu().to(torch.int64) & 0xFFFFFFFF
    on = ((b[..., None] >> torch.arange(32)) & 1).reshape(b.shape[0], -1)[:, :V]
    return [set(torch.nonzero(r)[:, 0].tolist()) for r in on]


@torch.no_grad()
@pytest.mark.parametrize("V", [32003, 1000])
@pytest.mark.parametrize("B", [1, 16, 64])
def test_kernel_matches_fp64_rules(V, B):
    rng = np.random.default_rng(7 * B + V)
    n_far = n_all = n_dec = 0
    for rep in range(6):
        T = [float(rng.choice([0.0, 1e-4, 0.2, 1.5])) for _ in range(B)]
        k = [int(rng.choice([0, 1, 50, V + 5])) for _ in range(B)]
        p = [float(rng.choice([0.0, 0.5, 0.9, 0.999, 1.0])) for _ in range(B)]
        r = [float(rng.choice([1.0, 0.8, 1.1, 1.3])) for _ in range(B)]
        kinds = [int(rng.integers(0, 3)) for _ in range(B)]
        sets = [set() if c == 0 else set(range(V)) if c == 2 else set(rng.choice(V, 300, replace=False).tolist())
                for c in kinds]
        x = _rows(B, V, rep * 131 + B, torch.tensor([6.0 * max(t, 0.2) for t in T]))
        seed = [int(rng.integers(0, 2 ** 63)) for _ in range(B)]
        ctr = [int(rng.integers(0, 2 ** 31)) for _ in range(B)]
        tset = _bits(sets, V)
        top_n = [20] * B
        tok, ids, lp = vn.op_sample_ex(x.to(DEV), T, k, seed, ctr, p, r, token_sets=tset, top_n=top_n)
        tok, ids = tok.cpu().tolist(), ids.cpu()
        after = _unbits(tset, V)
        # p = 1, r = 1: the 16-bit sampler's token and log-probs bit for bit
        t16, i16, l16 = vn.op_sample_logprobs(x.to(DEV), T, k, seed, ctr, top_n)
        plain = _unbits(_bits(sets, V), V)
        for b in range(B):
            assert after[b] == plain[b] | {tok[b]}, b
            xn = x[b].numpy()
            if p[b] == 1.0 and r[b] == 1.0:
                assert tok[b] == int(t16[b])
                assert torch.equal(ids[b], i16[b].cpu()) and torch.equal(lp[b].cpu().view(torch.int32),
                                                                          l16[b].cpu().view(torch.int32))
            u = float(R.uniform(seed[b], ctr[b]))
            want, keep, margin = N.choose(xn, T[b], k[b], p[b], r[b], sets[b], u)
            if T[b] == 0:
                xp = torch.from_numpy(N.penalize(xn, r[b], sets[b]))
                assert tok[b] == want == int(torch.argmax(xp)), (b, tok[b], want)
                continue
            if margin is None:
                continue
            assert keep[tok[b]], (b, T[b], k[b], p[b], r[b], tok[b])
            n_all += 1
            if margin >= 1e-5:
                n_far += 1
                assert tok[b] == want, (b, T[b], k[b], p[b], r[b], u, tok[b], want, margin)
            z = N.scaled(N.penalize(xn, r[b], sets[b]), T[b])
            _, margins = N.top_p_keep(z, N.topk_keep(z, k[b]), p[b])
            if N.decided(margins, 1e-6):
                n_dec += 1
                alt = [a for a in ids[b, 1:].tolist() if a >= 0]
                order = np.lexsort((np.arange(V), -np.where(keep, z, -np.inf)))
                assert alt == order[:min(20, int(keep.sum()))].tolist(), (b, alt[:5])
    assert n_all == 0 or n_far >= 0.999 * n_all - 1, (n_far, n_all)
    assert n_all == 0 or n_dec >= 0.5 * n_all, (n_dec, n_all)


@torch.no_grad()
def test_distribution_chi_square():
    from scipy.stats import chisquare
    V, N_ = 257, 20000
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(V, generator=g) * 2).bfloat16().float()
    toks = set(range(0, V, 3))
    T, k, p, r = 1.0, 0, 0.9, 1.3
    z = N.scaled(N.penalize(x.numpy(), r, toks), T)
    keep, _ = N.top_p_keep(z, N.topk_keep(z, k), p)
    w = np.where(keep, np.exp(z.astype(np.float64) - z[keep].max()), 0.0)
    prob = w / w.sum()
    xs = x[None].expand(N_, V).contiguous().to(DEV)
    tset = _bits([toks] * N_, V)
    tok = vn.op_sample_ex(xs, [T] * N_, [k] * N_, [12345] * N_, list(range(N_)), [p] * N_, [r] * N_,
                          token_sets=tset).cpu().numpy()
    assert keep[tok].all()
    cnt = np.bincount(tok, minlength=V)[keep]
    assert chisquare(cnt, prob[keep] * N_).pvalue > 1e-3


def _flat_model(max_batch=4):
    m = _model(SMALL, max_batch=max_batch)
    m.load_state_dict(to_dev(O.random_llm_state(SMALL, seed=21)))
    return m


def _gen(m, ids, vf, n, **kw):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=n, **kw)
    st.synchronize()
    return out


@torch.no_grad()
def test_token_sets_follow_the_sequence_and_greedy_penalty_is_the_penalized_argmax():
    m = _flat_model()
    ids = O.make_prompt_ids(SMALL, 356, seed=3, batch=3).to(DEV)
    vf = video_feats(3, 4)
    out = _gen(m, ids, vf, 12, repetition_penalty=1.3, eos_token_id=None)
    eng = m._engine
    for b in range(3):
        assert set(eng.read_token_set(b).tolist()) == set(out[b].tolist())
    # a continuation: the set is the whole conversation
    new = O.make_prompt_ids(SMALL, 0, seed=4, batch=3)[:, 1:9].to(DEV)
    out2 = m.generate_continue(new, max_new_tokens=8, repetition_penalty=1.3, eos_token_id=None)
    for b in range(3):
        assert set(eng.read_token_set(b).tolist()) == set(out2[b].tolist())
    # teacher-forced: the scored logits of every new position, penalized over the ids before it
    S = ids.shape[1]
    logits = m(out, video_spatio_temporal_features=vf, logits_to_keep=0).logits.float().cpu()
    checked = 0
    for b in range(3):
        for j in range(S, out.shape[1]):
            x = logits[b, j - 1].numpy()
            xp = N.penalize(x, 1.3, out[b, :j].tolist())
            top = np.sort(xp)[::-1][:2]
            if top[0] - top[1] > 3 * R.bf16_ulp(top[0]):
                checked += 1
                assert int(out[b, j]) == int(np.argmax(xp)), (b, j)
    assert checked >= 8
    # left-padded
    mask = torch.ones_like(ids)
    mask[1, :5] = 0
    pids = ids.clone()
    pids[1, :5] = 0
    out3 = _gen(m, pids, vf, 12, attention_mask=mask, do_sample=True, temperature=0.7, top_p=0.9, seed=3,
                repetition_penalty=1.2, eos_token_id=None)
    for b in range(3):
        assert set(eng.read_token_set(b).tolist()) == set(out3[b].tolist())


@torch.no_grad()
def test_default_after_penalized_equals_fresh_engine():
    ids = O.make_prompt_ids(SMALL, 356, seed=5, batch=2).to(DEV)
    vf = video_feats(2, 6)
    kw = dict(do_sample=True, temperature=0.7, top_k=50, seed=11, eos_token_id=None)
    fresh = _flat_model()
    a = _gen(fresh, ids, vf, 20, **kw)
    used = _flat_model()
    _gen(used, ids, vf, 20, top_p=0.8, repetition_penalty=1.2, **kw)
    _gen(used, ids, vf, 20, **kw)            # graphs of the default settings captured
    n0 = vn.launch_count()
    b = _gen(used, ids, vf, 20, **kw)
    lb = vn.launch_count() - n0
    n0 = vn.launch_count()
    _gen(fresh, ids, vf, 20, **kw)            # its default graphs were captured by the first call
    la = vn.launch_count() - n0
    assert torch.equal(a, b) and la == lb
    # greedy too
    g1 = _gen(fresh, ids, vf, 20, eos_token_id=None)
    g2 = _gen(used, ids, vf, 20, eos_token_id=None)
    assert torch.equal(g1, g2)


def _model_at(max_seq, kv_blocks=None, fmt="bf16", max_batch=4):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    c = VideoChatGPTConfig(hidden_size=SMALL.hidden, intermediate_size=SMALL.inter, num_hidden_layers=SMALL.layers,
                           num_attention_heads=SMALL.heads, vocab_size=SMALL.vocab, use_mm_proj=True,
                           mm_hidden_size=1024)
    clip = dict(hidden_size=1024, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=16)
    m = VideoChatGPTLlamaForCausalLM(c, clip_config=clip, max_batch=max_batch, max_seq=max_seq, kv_blocks=kv_blocks,
                                     llm_weight_format=fmt)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = 32000, 32001, 32002, True
    return m


def _run_requests(m, reqs, **kw):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        outs = m.generate_requests(reqs, eos_token_id=None, **kw)
    st.synchronize()
    return [o.cpu().tolist() for o in outs]


@torch.no_grad()
def test_requests_reproducible_across_slots_and_admission():
    m = _flat_model(max_batch=4)
    reqs = _requests(SMALL, [20, 5, 12, 7, 3, 10, 6], text_only=(3,))
    for i, r in enumerate(reqs):
        r.update(do_sample=i != 2, temperature=0.9, top_k=0, seed=17 * i, top_p=[0.9, 1.0, 0.5][i % 3],
                 repetition_penalty=[1.3, 1.0, 1.1, 0.8][i % 4])
    base = _run_requests(m, reqs, slots=3)
    assert _run_requests(m, reqs, slots=3) == base
    assert _run_requests(m, reqs, slots=1) == base
    assert _run_requests(m, reqs, slots=4, packed_admission=True) == base
    # each request alone through generate
    for i in (0, 2, 4):
        r = reqs[i]
        kw = dict(do_sample=r["do_sample"], temperature=0.9, top_k=0, seed=r["seed"], top_p=r["top_p"],
                  repetition_penalty=r["repetition_penalty"], eos_token_id=None)
        ids = torch.as_tensor(r["input_ids"]).reshape(1, -1).to(DEV)
        vf = r.get("video_spatio_temporal_features")
        out = _gen(m, ids, None if vf is None else vf[None].to(DEV), r["max_new_tokens"], **kw)
        assert out.cpu().tolist()[0] == base[i][0], i


@torch.no_grad()
def test_paged_preemption_reproducible():
    state = to_dev(O.random_llm_state(SMALL, seed=21))
    mc = _model_at(480)
    mc.load_state_dict(dict(state))
    mp = _model_at(480, kv_blocks=7)
    mp.load_state_dict(dict(state))
    # text prompts of ~50 tokens admitted with one block each grow to two: four slots need 8 of the 6 usable blocks
    reqs = _requests(SMALL, [150] * 5, text_only=(0, 1, 2, 3, 4))
    for i, r in enumerate(reqs):
        r.update(do_sample=True, temperature=1.0, top_k=0, seed=5 + i, top_p=0.95, repetition_penalty=1.2)
    want = _run_requests(mc, reqs, slots=4)
    got = _run_requests(mp, reqs, slots=4)
    assert mp.last_kv_stats["preemptions"] > 0
    assert got == want
    assert _run_requests(mp, reqs, slots=4, packed_admission=True) == want


def test_abi_rejections():
    m = _flat_model()
    eng = m._ensure_engine(need_llm=True)
    bad = [dict(top_p=[1.5]), dict(top_p=[float("nan")]), dict(top_p=[-0.1]), dict(repetition_penalty=[0.0]),
           dict(repetition_penalty=[float("inf")]), dict(repetition_penalty=[-2.0])]
    for kw in bad:
        args = dict(top_p=[1.0], repetition_penalty=[1.0])
        args.update(kw)
        with pytest.raises(vn.VclError):
            eng.set_sampling_ex([0], [1.0], [0], [1], args["top_p"], args["repetition_penalty"])
    with pytest.raises(vn.VclError, match="twice"):
        eng.set_sampling_ex([1, 1], [1.0, 1.0], [0, 0], [1, 2], [0.9, 0.9], [1.0, 1.0])
    with pytest.raises(vn.VclError):
        eng.set_sampling_ex([99], [1.0], [0], [1], [0.9], [1.0])
    with pytest.raises(vn.VclError):
        eng.set_token_set(99, [1, 2])
    x = torch.zeros(1, vn.SAMPLE_WIDE_MAX_V + 1, device=DEV)
    with pytest.raises(vn.VclError, match="outside"):
        vn.op_sample_ex(x, [1.0], [0], [1], [0], [0.9], [1.0])
    with pytest.raises(vn.VclError):
        vn.op_sample_ex(x[:, :100].contiguous(), [1.0], [0], [1], [0], [1.2], [1.0])


@torch.no_grad()
def test_sessions_and_chunked_prompts_keep_their_token_sets():
    """On a paged model: the set after a session's first turn and after its continuation is the whole conversation;
    after a chunked prompt it is the prompt and its tokens (no token a discarded chunk draw left behind); and a chunked,
    penalized, top-p request returns what generate returns for it on a contiguous model (one-shot prefill)."""
    state = to_dev(O.random_llm_state(SMALL, seed=21))
    mp = _model_at(1024, kv_blocks=20)
    mp.load_state_dict(dict(state))
    mc = _model_at(1024)
    mc.load_state_dict(dict(state))
    samp = dict(do_sample=True, temperature=0.9, top_k=0, top_p=0.9, repetition_penalty=1.3)
    # 9 new tokens: the prefill's and one decode chunk of 8, so the slot decodes nothing past the request
    g = torch.Generator().manual_seed(8)
    first = torch.cat([torch.tensor([1]), torch.randint(3, 32000, (39,), generator=g)])
    out1 = _run_requests(mp, [dict(input_ids=first, max_new_tokens=9, seed=3, session="a", **samp)], slots=1)[0][0]
    eng = mp._engine
    assert set(eng.read_token_set(0).tolist()) == set(out1)
    turn = torch.randint(3, 32000, (10,), generator=g)
    out2 = _run_requests(mp, [dict(input_ids=turn, max_new_tokens=9, seed=4, continues="a", **samp)], slots=1)[0][0]
    assert out2[:len(out1) + 10] == out1 + turn.tolist()
    assert set(eng.read_token_set(0).tolist()) == set(out2)
    mp.end_session()
    # a 700-token prompt in two chunks (512 + 188)
    long = torch.cat([torch.tensor([1]), torch.randint(3, 32000, (699,), generator=g)])
    req = dict(input_ids=long, max_new_tokens=9, seed=5, **samp)
    got = _run_requests(mp, [req], slots=1, chunked_prefill=True)[0][0]
    assert mp.last_kv_stats["chunk_calls"] == 2
    assert set(eng.read_token_set(0).tolist()) == set(got)
    want = _gen(mc, long[None].to(DEV), None, 9, seed=5, eos_token_id=None, **samp)
    assert got == want.cpu().tolist()[0]
    # chunked next to short prompts, packed: the same tokens
    reqs = [req, dict(input_ids=first, max_new_tokens=20, seed=6, **samp),
            dict(input_ids=long[:600], max_new_tokens=12, seed=7, **samp)]
    base = _run_requests(mp, reqs, slots=3, chunked_prefill=True)
    assert base[0][0] == got
    assert _run_requests(mp, reqs, slots=3, chunked_prefill=True, packed_admission=True) == base
    assert _run_requests(mp, reqs, slots=1, chunked_prefill=True) == base


# ---- end to end: HF's processors on the bf16 oracle's logits ---------------------------------------------------------
ET, EP, ER = 0.7, 0.9, 1.3        # temperature, top_p, repetition_penalty of the end-to-end tests (top_k 0)


def _hf_choice(x, before, u):
    """HF's RepetitionPenalty / Temperature / TopP processors on logits x [V] fp32 after the ids `before`, then the
    device's draw (first index whose inclusive prefix sum of the kept weights exceeds u * W) -> (token, kept)"""
    from transformers.generation.logits_process import (RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                        TopPLogitsWarper)
    ids = before[None]
    s = RepetitionPenaltyLogitsProcessor(penalty=ER)(ids, x[None].clone())
    s = TopPLogitsWarper(top_p=EP)(ids, TemperatureLogitsWarper(ET)(ids, s))[0].double()
    kept = torch.isfinite(s)
    w = torch.where(kept, torch.exp(s - s[kept].max()), torch.zeros_like(s))
    c = torch.cumsum(w, 0)
    j = int(torch.nonzero((c > u * c[-1]) & (w > 0))[0])
    return j, kept


def _decided(x, before, u, ulps=3):
    """HF's choice, and whether it holds when the logits move by `ulps` bf16 ulps in the two directions that move the
    chosen interval's edges furthest (the kept set unchanged too)"""
    j, kept = _hf_choice(x, before, u)
    d = torch.from_numpy(ulps * R.bf16_ulp(x.numpy())).float()
    idx = torch.arange(x.numel())
    for sgn in (torch.where(idx < j, 1.0, -1.0), torch.where(idx <= j, -1.0, 1.0)):
        j2, k2 = _hf_choice(x + d * sgn, before, u)
        if j2 != j or not torch.equal(k2, kept):
            return j, False
    return j, True


def _check_e2e(toks, o_logits, prompts, seeds, counters0, what, tally):
    """toks [B, n] engine tokens, o_logits [n, B, V] the oracle teacher-forced with them, prompts [B] the ids before
    the first new token of each row"""
    B, n = toks.shape
    for b in range(B):
        for i in range(n):
            before = torch.cat([prompts[b].cpu(), toks[b, :i].cpu()]).long()
            u = float(R.uniform(seeds[b], counters0[b] + i))
            j, ok = _decided(o_logits[i, b].float().cpu(), before, u)
            tally[1] += 1
            if ok:
                tally[0] += 1
                assert int(toks[b, i]) == j, (what, b, i, int(toks[b, i]), j)


@pytest.fixture(scope="module")
def e2e_tally():
    t = [0, 0]
    yield t
    print(f"[nucleus] end-to-end margin rule: {t[0]}/{t[1]} steps decided")


@torch.no_grad()
@pytest.mark.parametrize("fmt", ["bf16", "fp8_e4m3"])
def test_end_to_end_matches_hf_processors_where_decided(fmt, e2e_tally):
    """generate, generate_continue and generate_requests sample with top_p and the penalty from the handle's table,
    inside the captured graphs; at every decided step the token is the one HF's processors on the bf16 oracle's
    logits give for the same u (fp8: the oracle runs on the dequantized weights W~ the engine computes with)"""
    from test_sampling_gpu import peaked_state
    import _fp8_ref as F8
    sd = to_dev(peaked_state())
    osd = sd if fmt == "bf16" else F8.dequantize_state(sd)
    m = _model_at(480, fmt=fmt)
    m.load_state_dict(dict(sd))
    kw = dict(do_sample=True, temperature=ET, top_k=0, top_p=EP, repetition_penalty=ER, eos_token_id=None)
    B, n, seed = 3, 10, 900
    ids = O.make_prompt_ids(SMALL, 356, seed=61, batch=B).to(DEV)
    vf = video_feats(B, 62)
    S = ids.shape[1]
    out = _gen(m, ids, vf, n, seed=seed, **kw)
    toks = out[:, S:]
    _, o_logits = O.greedy_generate(osd, SMALL, ids, vf.bfloat16(), n, forced=toks)
    _check_e2e(toks, o_logits, list(ids), [seed + b for b in range(B)], [S] * B, f"{fmt} generate", e2e_tally)
    # the next turn: the set is the whole conversation, the first new token takes position L
    new = O.make_prompt_ids(SMALL, 0, seed=63, batch=B)[:, 1:7].to(DEV)
    ctx = torch.cat([out, new], 1)
    L = ctx.shape[1]
    out2 = m.generate_continue(new, max_new_tokens=8, seed=seed + 50, **kw)
    toks2 = out2[:, L:]
    _, o2 = O.greedy_generate(osd, SMALL, ctx, vf.bfloat16(), toks2.shape[1], forced=toks2)
    _check_e2e(toks2, o2, list(ctx), [seed + 50 + b for b in range(B)], [L] * B, f"{fmt} continue", e2e_tally)
    # in flight, next to each other
    reqs = _requests(SMALL, [9, 12, 7], text_only=(1,))
    for i, r in enumerate(reqs):
        r.update(seed=1000 + i, **{k: v for k, v in kw.items() if k != "eos_token_id"})
    outs = _run_requests(m, reqs, slots=2)
    for i, r in enumerate(reqs):
        p = torch.as_tensor(r["input_ids"]).reshape(-1).to(DEV)
        f = r.get("video_spatio_temporal_features")
        f = None if f is None else f[None].to(DEV).bfloat16()
        t = torch.tensor(outs[i][0][p.numel():], device=DEV)[None]
        _, o3 = O.greedy_generate(osd, SMALL, p[None], f, t.shape[1], forced=t)
        _check_e2e(t, o3, [p], [1000 + i], [p.numel()], f"{fmt} request {i}", e2e_tally)


def test_most_end_to_end_steps_are_decided(e2e_tally):
    assert e2e_tally[1] > 0 and e2e_tally[0] >= 0.5 * e2e_tally[1], e2e_tally

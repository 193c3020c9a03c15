"""Min-p, typical, epsilon and eta warpers on the GPU (sampling.cu's warp_row, vcl_llm_set_warpers).

Bars:
- the kernel against the float64 rules of _warpers_ref.py over V 32 003 / 1 000, B 1 / 16 / 64, T 0.2 / 0.7 / 1.5,
  top-k 0 / 50, top-p 1 / 0.9 and every warper alone and all four together, rows where typical drops the arg-max
  included: the token is always in the fp64 final set and is the fp64 choice wherever u * W lies at least 1e-5 W from
  its interval's edges; on decided rows the log-prob alternatives are the final set's largest tokens and the chosen
  token's log-prob is within 1e-5 + 2^-22 |lp| of the fp64 value;
- with all four off, tokens and log-probs equal vcl_op_sample_ex's bit for bit;
- a chi-square test of one row with all four warpers against its exact probabilities;
- the graph loops: seeded generate's tokens equal vcl_op_sample_warpers on decode_step's logits, teacher-forced, bit
  for bit (plain, left-padded, generate_continue, and guided, whose rows vcl_op_guidance combines first); guided
  unseeded sampling equals a replay of HF's guidance and the host warpers with torch's RNG;
- fp8: an fp8 engine's tokens equal a bf16 engine's on the dequantized weights W~, bit for bit;
- end to end: at every step that a 3-ulp move of the logits cannot change, the token of generate, generate_continue
  and generate_requests (all four warpers, T 0.7) is the one HF's own warpers on the bf16 oracle's logits give for the
  same u, on bf16 and fp8 engines; at least half the steps are decided;
- in flight: a request's tokens equal generate's for it alone, across slots, admission modes, paging and preemption;
- a default call after a warper call equals a fresh engine's, with the same launch count; the C ABI rejections.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
import _nucleus_ref as N  # noqa: E402
import _sampling_ref as R  # noqa: E402
import _warpers_ref as Wr  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import to_dev  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402
from test_inflight_gpu import _model, _requests  # noqa: E402
from test_nucleus_gpu import _model_at, _run_requests  # noqa: E402

DEV = "cuda"
SMALL = O.LlmCfg(hidden=512, inter=1024, heads=4, layers=2)
SETTINGS = [(0.05, 1.0, 0.0, 0.0), (1.0, 1.0, 0.0, 0.0), (0.0, 0.2, 0.0, 0.0), (0.0, 0.9, 0.0, 0.0),
            (0.0, 0.999, 0.0, 0.0), (0.0, 1.0, 3e-4, 0.0), (0.0, 1.0, 3e-2, 0.0), (0.0, 1.0, 0.0, 3e-4),
            (0.0, 1.0, 0.0, 3e-2), (0.05, 0.9, 3e-4, 3e-4), Wr.OFF]


def _rows(B, V, rng, T):
    """logits rows (bf16 values): normal rows of spread 6 T, and every third one a peaked row, a near-flat row with one
    token of probability ~0.3, on which typical at small mass drops the arg-max"""
    x = (torch.from_numpy(rng.standard_normal((B, V))) * torch.tensor([6.0 * t for t in T])[:, None]).float()
    for b in range(0, B, 3):
        x[b] = torch.from_numpy(rng.standard_normal(V) * 0.05 * T[b]).float()
        x[b, int(rng.integers(0, V))] = math.log(0.43 * V) * T[b]
    return x.bfloat16().float()


@torch.no_grad()
@pytest.mark.parametrize("V", [32003, 1000])
@pytest.mark.parametrize("B", [1, 16, 64])
def test_kernel_matches_fp64_rules(V, B):
    rng = np.random.default_rng(11 * B + V)
    n_all = n_far = n_dec = n_drop_max = 0
    for rep in range(4 if B > 1 else 24):
        T = [float(rng.choice([0.2, 0.7, 1.5])) for _ in range(B)]
        k = [int(rng.choice([0, 50])) for _ in range(B)]
        p = [float(rng.choice([1.0, 0.9])) for _ in range(B)]
        ws = [SETTINGS[int(rng.integers(0, len(SETTINGS)))] for _ in range(B)]
        x = _rows(B, V, rng, T)
        seed = [int(rng.integers(0, 2 ** 63)) for _ in range(B)]
        ctr = [int(rng.integers(0, 2 ** 31)) for _ in range(B)]
        cols = list(zip(*ws))
        tok, ids, lp = vn.op_sample_warpers(x.to(DEV), T, k, seed, ctr, p, [1.0] * B, *cols, top_n=[20] * B)
        tok, ids, lp = tok.cpu().tolist(), ids.cpu(), lp.cpu()
        t0, i0, l0 = vn.op_sample_ex(x.to(DEV), T, k, seed, ctr, p, [1.0] * B, top_n=[20] * B)
        for b in range(B):
            if ws[b] == Wr.OFF:     # all four off: vcl_op_sample_ex bit for bit
                assert tok[b] == int(t0[b])
                assert torch.equal(ids[b], i0[b].cpu())
                assert torch.equal(lp[b].view(torch.int32), l0[b].cpu().view(torch.int32))
            xn = x[b].numpy()
            u = float(R.uniform(seed[b], ctr[b]))
            want, kept, zmax, m, margin = Wr.choose(xn, T[b], k[b], p[b], ws[b], u)
            z = N.scaled(xn, T[b])
            n_all += 1
            dec = Wr.decided(m, 1e-5, 1e-5)
            if dec:
                assert kept[tok[b]], (b, T[b], k[b], p[b], ws[b], tok[b])
            if dec and margin >= 1e-5:
                n_far += 1
                assert tok[b] == want, (b, T[b], k[b], p[b], ws[b], tok[b], want, margin)
            if dec:
                n_dec += 1
                n_drop_max += not kept[int(np.argmax(z))]
                alt = [a for a in ids[b, 1:].tolist() if a >= 0]
                order = np.lexsort((np.arange(V), -np.where(kept, z, -np.inf)))
                assert alt == order[:min(20, int(kept.sum()))].tolist(), (b, ws[b], alt[:5])
                ref = Wr.logprob(z, kept, zmax, tok[b])
                assert abs(float(lp[b, 0]) - ref) <= 1e-5 + 2 ** -22 * abs(ref), (b, ws[b], float(lp[b, 0]), ref)
    print(f"V={V} B={B}: {n_dec} of {n_all} rows decided, {n_far} draws decided, {n_drop_max} drop the arg-max")
    assert n_dec >= 0.5 * n_all, (n_dec, n_all)
    # (a near-flat row keeps thousands of tokens, whose intervals are narrower than 1e-4 of W')
    assert n_far >= 0.5 * n_dec, (n_far, n_dec)
    if V == 32003 and B > 1:
        assert n_drop_max > 0


@torch.no_grad()
def test_distribution_chi_square():
    from scipy.stats import chisquare
    V, N_ = 257, 20000
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(V, generator=g) * 2).bfloat16().float()
    T, k, p, w = 1.0, 0, 1.0, (0.02, 0.95, 1e-3, 1e-3)
    z = N.scaled(x.numpy(), T)
    kept, zmax, m = Wr.warp_keep(z, N.topk_keep(z, k), w)
    assert Wr.decided(m, 1e-4, 1e-4), m
    wt = np.where(kept, np.exp(z.astype(np.float64) - float(zmax)), 0.0)
    prob = wt / wt.sum()
    xs = x[None].expand(N_, V).contiguous().to(DEV)
    tok = vn.op_sample_warpers(xs, [T] * N_, [k] * N_, [12345] * N_, list(range(N_)), [p] * N_, [1.0] * N_,
                               *[[v] * N_ for v in w]).cpu().numpy()
    assert kept[tok].all()
    cnt = np.bincount(tok, minlength=V)[kept]
    assert chisquare(cnt, prob[kept] * N_).pvalue > 1e-3


def _flat_model(max_batch=4, max_seq=None):
    m = _model(SMALL, max_batch=max_batch) if max_seq is None else _model_at(max_seq, max_batch=max_batch)
    m.load_state_dict(to_dev(O.random_llm_state(SMALL, seed=21)))
    return m


def _gen(m, ids, vf, n, **kw):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        out = m.generate(ids, video_spatio_temporal_features=vf, max_new_tokens=n, **kw)
    st.synchronize()
    return out


WARP_KW = dict(min_p=0.05, typical_p=0.9, epsilon_cutoff=3e-4, eta_cutoff=3e-4)


def _teacher_forced(eng, logits, S, n, T, k, seed, warp, B, pads=None):
    """tokens of n steps: vcl_op_sample_warpers on each step's logits (row b at seed + b, counter = its position,
    the cache column less its left padding), each token fed back through decode_step"""
    toks, pos = [], S
    pads = pads or [0] * B
    for step in range(n):
        t = vn.op_sample_warpers(logits, [T] * B, [k] * B, [seed + b for b in range(B)], [pos - p for p in pads],
                                 [1.0] * B, [1.0] * B, *[[v] * B for v in warp])
        toks.append(t.to(torch.int64))
        if step + 1 == n:
            break
        logits, _ = eng.decode_step(t, pos, want_logits=True)
        pos += 1
    return torch.stack(toks, dim=1)


@torch.no_grad()
@pytest.mark.parametrize("kw", [dict(min_p=0.05), dict(typical_p=0.5), dict(epsilon_cutoff=3e-2),
                                dict(eta_cutoff=3e-2), WARP_KW])
def test_graph_loop_equals_the_op_teacher_forced(kw):
    m = _flat_model()
    B, n, T, k, seed = 2, 12, 1.5, 0, 77
    ids = O.make_prompt_ids(SMALL, 356, seed=5, batch=B).to(DEV)     # (356 video rows)
    S = ids.shape[1]
    vf = video_feats(B, 6)
    out = _gen(m, ids, vf, n, do_sample=True, temperature=T, top_k=k, seed=seed, eos_token_id=None, **kw)
    warp = m._warper_args(kw.get("min_p"), kw.get("typical_p"), kw.get("epsilon_cutoff"), kw.get("eta_cutoff"))
    eng = m._ensure_engine(need_llm=True)
    vs = m._spans_dev(ids, vf, eng.NV)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        _, logits, _ = eng.prefill(ids, vf.cuda(), vs, want_logits=True, want_token=False)
        want = _teacher_forced(eng, logits, S, n, T, k, seed, warp, B)
    st.synchronize()
    assert torch.equal(out[:, S:].cpu(), want.cpu())
    # generate_continue: the next turn's tokens, the same way
    new = O.make_prompt_ids(SMALL, 6, seed=8, batch=B)[:, -6:].to(DEV)
    with torch.cuda.stream(st):
        out2 = m.generate_continue(new, do_sample=True, temperature=T, top_k=k, seed=seed + 1, max_new_tokens=n,
                                   eos_token_id=None, **kw)
    st.synchronize()
    ctx = torch.cat([out, new], dim=1)
    with torch.cuda.stream(st):
        tail = torch.cat([out[:, -1:], new], dim=1)
        _, logits, _ = eng.prefill_append(tail, S + n - 1, want_logits=True, want_token=False)
        want2 = _teacher_forced(eng, logits, ctx.shape[1], n, T, k, seed + 1, warp, B)
    st.synchronize()
    assert torch.equal(out2[:, ctx.shape[1]:].cpu(), want2.cpu())


@torch.no_grad()
@pytest.mark.parametrize("kw", [dict(typical_p=0.5), WARP_KW])
def test_padded_graph_loop_equals_the_op_teacher_forced(kw):
    from test_padded_batch_gpu import padded_batch
    m = _flat_model()
    ids, pads, _ = padded_batch(SMALL, [10, 25, 3], seed=8)
    B, S, n, T, k, seed = 3, ids.shape[1], 12, 1.5, 0, 41
    mask = (torch.arange(S)[None] >= torch.tensor(pads)[:, None]).long().to(DEV)
    vf = video_feats(B, 9)
    out = _gen(m, ids, vf, n, attention_mask=mask, do_sample=True, temperature=T, top_k=k, seed=seed,
               eos_token_id=None, **kw)
    warp = m._warper_args(*[kw.get(x) for x in ("min_p", "typical_p", "epsilon_cutoff", "eta_cutoff")])
    eng = m._ensure_engine(need_llm=True)
    vs = m._spans_dev(ids, vf, eng.NV, pads)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        _, logits, _ = eng.prefill(ids, vf, vs, want_logits=True, want_token=False, n_pad=pads)
        want = _teacher_forced(eng, logits, S, n, T, k, seed, warp, B, pads)
    st.synchronize()
    assert torch.equal(out[:, S:].cpu(), want.cpu())


def _guided(m, n, **kw):
    ids = O.make_prompt_ids(SMALL, 356, seed=31, batch=1).to(DEV)
    vf = video_feats(1, 32)
    neg = torch.cat([torch.tensor([1]), torch.randint(3, 32000, (39,), generator=torch.Generator().manual_seed(33))])
    neg = neg[None].to(DEV)
    return ids, vf, neg, _gen(m, ids, vf, n, eos_token_id=None, guidance_scale=1.75, negative_prompt_ids=neg, **kw)


@torch.no_grad()
def test_guided_seeded_graph_loop_equals_the_ops():
    """guided seeded generate (the warpers after the guidance, on the device) against decode_step's raw logits of both
    clips, combined by vcl_op_guidance and drawn by vcl_op_sample_warpers"""
    g, n, T, k, seed = 1.75, 12, 1.5, 0, 5
    m = _flat_model()
    ids, vf, neg, out = _guided(m, n, do_sample=True, temperature=T, top_k=k, seed=seed, **WARP_KW)
    S = ids.shape[1]
    toks = out[0, S:].tolist()
    warp = m._warper_args(*[WARP_KW[x] for x in ("min_p", "typical_p", "epsilon_cutoff", "eta_cutoff")])
    eng = m._engine
    ids2, pads2, spans, f2, shift = m._guided_batch(ids, None, vf, neg, None, None, eng.NV)
    assert shift == 0
    eng.set_guidance([0, 1], [1, -1], [g, 1.0])
    plain = 0
    try:
        _, logits, _ = eng.prefill(ids2, f2, spans, want_logits=True, n_pad=pads2)
        for i in range(n):
            comb = vn.op_guidance(logits, [1, -1], [g, 1.0])[:1].contiguous()
            want = int(vn.op_sample_warpers(comb, [T], [k], [seed], [S + i], [1.0], [1.0], *[[v] for v in warp])[0])
            plain += want != int(vn.op_sample_ex(comb, [T], [k], [seed], [S + i], [1.0], [1.0])[0])
            assert toks[i] == want, i
            if i + 1 < n:
                logits, _ = eng.decode_step(torch.tensor([want, want], dtype=torch.int32, device=DEV), S + i,
                                            want_logits=True)
    finally:
        eng.set_guidance([0, 1], [-1, -1], [1.0, 1.0])
    assert plain > 0          # the warpers changed some draw


@torch.no_grad()
def test_guided_unseeded_applies_the_host_warpers():
    """guided unseeded sampling (the stepwise path: HF's guidance, then the processors and the warpers on the host)
    against a replay of that chain with torch's RNG from the same seed"""
    from video_chatgpt.model import VideoChatGPTLlamaForCausalLM as M
    g, n, T, k = 1.75, 10, 1.5, 0
    m = _flat_model()
    warp = m._warper_args(*[WARP_KW[x] for x in ("min_p", "typical_p", "epsilon_cutoff", "eta_cutoff")])
    torch.manual_seed(123)
    ids, vf, neg, out = _guided(m, n, do_sample=True, temperature=T, top_k=k, **WARP_KW)
    S = ids.shape[1]
    eng = m._engine
    ids2, pads2, spans, f2, _ = m._guided_batch(ids, None, vf, neg, None, None, eng.NV)
    torch.manual_seed(123)
    st = torch.cuda.Stream()
    seq, shrunk = ids.clone(), 0
    with torch.cuda.stream(st):
        _, logits, _ = eng.prefill(ids2, f2, spans, want_logits=True, want_token=False, n_pad=pads2)
        pos = ids2.shape[1]
        for i in range(n):
            comb = M._host_guidance(logits[:1], logits[1:], g)
            lg = M._host_processors(seq, comb, True, T, k, 1.0, 1.0, None, S, warp)
            shrunk += int(torch.isfinite(lg).sum()) < int(torch.isfinite(comb).sum())
            nxt = torch.multinomial(torch.softmax(lg, dim=-1), 1)[:, 0]
            seq = torch.cat([seq, nxt[:, None].to(torch.int64)], dim=1)
            if i + 1 < n:
                feed = nxt.to(torch.int32)
                logits, _ = eng.decode_step(torch.cat([feed, feed]).contiguous(), pos, want_logits=True)
                pos += 1
    st.synchronize()
    assert torch.equal(out.cpu(), seq.cpu())
    assert shrunk == n        # the warpers removed tokens at every step


@torch.no_grad()
def test_fp8_equals_bf16_on_dequantized_weights():
    """an fp8 engine with the warpers gives the tokens of a bf16 engine on the dequantized weights W~, bit for bit"""
    import _fp8_ref as F8
    sd = to_dev(O.random_llm_state(SMALL, seed=21))
    m8, mb = _model_at(480, fmt="fp8_e4m3"), _model_at(480)
    m8.load_state_dict(dict(sd))
    mb.load_state_dict(F8.dequantize_state(sd))
    ids = O.make_prompt_ids(SMALL, 356, seed=5, batch=2).to(DEV)
    vf = video_feats(2, 6)
    kw = dict(do_sample=True, temperature=1.5, top_k=0, seed=19, eos_token_id=None, **WARP_KW)
    a, b = _gen(m8, ids, vf, 16, **kw), _gen(mb, ids, vf, 16, **kw)
    assert torch.equal(a, b)
    reqs = _requests(SMALL, [9, 12, 7], text_only=(1,))
    for i, r in enumerate(reqs):
        r.update(do_sample=True, temperature=1.5, top_k=0, seed=70 + i, **WARP_KW)
    assert _run_requests(m8, reqs, slots=2) == _run_requests(mb, reqs, slots=2)


@torch.no_grad()
def test_default_after_warpers_equals_fresh_engine():
    ids = O.make_prompt_ids(SMALL, 356, seed=5, batch=2).to(DEV)
    vf = video_feats(2, 6)
    kw = dict(do_sample=True, temperature=0.7, top_k=50, seed=11, eos_token_id=None)
    fresh = _flat_model()
    a = _gen(fresh, ids, vf, 20, **kw)
    used = _flat_model()
    w = _gen(used, ids, vf, 20, **kw, **WARP_KW)
    _gen(used, ids, vf, 20, **kw)
    n0 = vn.launch_count()
    b = _gen(used, ids, vf, 20, **kw)
    lb = vn.launch_count() - n0
    n0 = vn.launch_count()
    _gen(fresh, ids, vf, 20, **kw)
    la = vn.launch_count() - n0
    assert torch.equal(a, b) and la == lb
    assert not torch.equal(a, w)            # the warpers did act
    g1 = _gen(fresh, ids, vf, 20, eos_token_id=None)
    g2 = _gen(used, ids, vf, 20, eos_token_id=None, **WARP_KW)   # greedy ignores them
    assert torch.equal(g1, g2)


@torch.no_grad()
def test_requests_reproducible_across_slots_and_admission():
    m = _flat_model(max_batch=4)
    reqs = _requests(SMALL, [20, 5, 12, 7, 3, 10, 6], text_only=(3,))
    opts = [dict(min_p=0.1), dict(typical_p=0.5), dict(), dict(epsilon_cutoff=3e-2, eta_cutoff=3e-2), WARP_KW]
    for i, r in enumerate(reqs):
        r.update(do_sample=True, temperature=1.5, top_k=0, seed=17 * i, **opts[i % len(opts)])
    base = _run_requests(m, reqs, slots=3)
    assert _run_requests(m, reqs, slots=1) == base
    assert _run_requests(m, reqs, slots=4, packed_admission=True) == base
    for i in (0, 1, 3, 4):
        r = reqs[i]
        ids = torch.as_tensor(r["input_ids"]).reshape(1, -1).to(DEV)
        vf = r.get("video_spatio_temporal_features")
        out = _gen(m, ids, None if vf is None else vf[None].to(DEV), r["max_new_tokens"], do_sample=True,
                   temperature=1.5, top_k=0, seed=r["seed"], eos_token_id=None, **opts[i % len(opts)])
        assert out.cpu().tolist()[0] == base[i][0], i


@torch.no_grad()
def test_paged_preemption_reproducible():
    state = to_dev(O.random_llm_state(SMALL, seed=21))
    mc = _model_at(480)
    mc.load_state_dict(dict(state))
    mp = _model_at(480, kv_blocks=7)
    mp.load_state_dict(dict(state))
    reqs = _requests(SMALL, [150] * 5, text_only=(0, 1, 2, 3, 4))
    for i, r in enumerate(reqs):
        r.update(do_sample=True, temperature=1.5, top_k=0, seed=5 + i, min_p=0.05 * (i % 2), typical_p=0.8)
    want = _run_requests(mc, reqs, slots=4)
    got = _run_requests(mp, reqs, slots=4)
    assert mp.last_kv_stats["preemptions"] > 0
    assert got == want
    assert _run_requests(mp, reqs, slots=4, packed_admission=True) == want


def test_abi_rejections():
    m = _flat_model()
    eng = m._ensure_engine(need_llm=True)
    for bad in ([1.5, 1.0, 0.0, 0.0], [float("nan"), 1.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0], [0.0, 1.5, 0.0, 0.0],
                [0.0, 1.0, 1.0, 0.0], [0.0, 1.0, -0.1, 0.0], [0.0, 1.0, 0.0, 1.0], [0.0, 1.0, 0.0, float("nan")]):
        with pytest.raises(vn.VclError, match="has to be"):
            eng.set_warpers([0], *[[v] for v in bad])
    with pytest.raises(vn.VclError, match="twice"):
        eng.set_warpers([1, 1], [0.1, 0.1], [1.0, 1.0], [0.0, 0.0], [0.0, 0.0])
    with pytest.raises(vn.VclError):
        eng.set_warpers([99], [0.1], [1.0], [0.0], [0.0])
    x = torch.zeros(1, vn.SAMPLE_WIDE_MAX_V + 1, device=DEV)
    with pytest.raises(vn.VclError, match="outside"):
        vn.op_sample_warpers(x, [1.0], [0], [1], [0], [1.0], [1.0], [0.1], [1.0], [0.0], [0.0])
    with pytest.raises(vn.VclError, match="min_p"):
        vn.op_sample_warpers(x[:, :100].contiguous(), [1.0], [0], [1], [0], [1.0], [1.0], [2.0], [1.0], [0.0], [0.0])


# ---- end to end: HF's warpers on the bf16 oracle's logits -----------------------------------------------------------
ET = 0.7                          # temperature of the end-to-end tests (top_k 0), with WARP_KW


def _hf_choice(x, u):
    """HF's Temperature / MinP / Typical / Epsilon / Eta warpers on logits x [V] fp32, then the device's draw (first
    index whose inclusive prefix sum of the kept weights exceeds u * W) -> (token, kept)"""
    from transformers.generation.logits_process import (EpsilonLogitsWarper, EtaLogitsWarper, MinPLogitsWarper,
                                                        TemperatureLogitsWarper, TypicalLogitsWarper)
    ids = torch.zeros(1, 1, dtype=torch.long)
    s = TemperatureLogitsWarper(ET)(ids, x[None].clone())
    for proc in (MinPLogitsWarper(min_p=WARP_KW["min_p"]), TypicalLogitsWarper(mass=WARP_KW["typical_p"]),
                 EpsilonLogitsWarper(epsilon=WARP_KW["epsilon_cutoff"]), EtaLogitsWarper(epsilon=WARP_KW["eta_cutoff"])):
        s = proc(ids, s)
    s = s[0].double()
    kept = torch.isfinite(s)
    w = torch.where(kept, torch.exp(s - s[kept].max()), torch.zeros_like(s))
    c = torch.cumsum(w, 0)
    return int(torch.nonzero((c > u * c[-1]) & (w > 0))[0]), kept


def _decided(x, u, ulps=3):
    """HF's choice, and whether it holds when the logits move by `ulps` bf16 ulps in the two directions that move the
    chosen interval's edges furthest (the kept set unchanged too) -- test_nucleus_gpu.py's rule"""
    j, kept = _hf_choice(x, u)
    d = torch.from_numpy(ulps * R.bf16_ulp(x.numpy())).float()
    idx = torch.arange(x.numel())
    for sgn in (torch.where(idx < j, 1.0, -1.0), torch.where(idx <= j, -1.0, 1.0)):
        j2, k2 = _hf_choice(x + d * sgn, u)
        if j2 != j or not torch.equal(k2, kept):
            return j, False
    return j, True


def _check_e2e(toks, o_logits, seeds, counters0, what, tally):
    B, n = toks.shape
    for b in range(B):
        for i in range(n):
            u = float(R.uniform(seeds[b], counters0[b] + i))
            j, ok = _decided(o_logits[i, b].float().cpu(), u)
            tally[1] += 1
            if ok:
                tally[0] += 1
                assert int(toks[b, i]) == j, (what, b, i, int(toks[b, i]), j)


@pytest.fixture(scope="module")
def e2e_tally():
    t = [0, 0]
    yield t
    print(f"[warpers] end-to-end margin rule: {t[0]}/{t[1]} steps decided")


@torch.no_grad()
@pytest.mark.parametrize("fmt", ["bf16", "fp8_e4m3"])
def test_end_to_end_matches_hf_warpers_where_decided(fmt, e2e_tally):
    """generate, generate_continue and generate_requests sample with all four warpers from the handle's table, inside
    the captured graphs; at every decided step the token is the one HF's warpers on the bf16 oracle's logits give for
    the same u (fp8: the oracle runs on the dequantized weights W~ the engine computes with)"""
    from test_sampling_gpu import peaked_state
    import _fp8_ref as F8
    sd = to_dev(peaked_state())
    osd = sd if fmt == "bf16" else F8.dequantize_state(sd)
    m = _model_at(480, fmt=fmt)
    m.load_state_dict(dict(sd))
    kw = dict(do_sample=True, temperature=ET, top_k=0, eos_token_id=None, **WARP_KW)
    B, n, seed = 3, 10, 900
    ids = O.make_prompt_ids(SMALL, 356, seed=61, batch=B).to(DEV)
    vf = video_feats(B, 62)
    S = ids.shape[1]
    out = _gen(m, ids, vf, n, seed=seed, **kw)
    toks = out[:, S:]
    _, o_logits = O.greedy_generate(osd, SMALL, ids, vf.bfloat16(), n, forced=toks)
    _check_e2e(toks, o_logits, [seed + b for b in range(B)], [S] * B, f"{fmt} generate", e2e_tally)
    new = O.make_prompt_ids(SMALL, 0, seed=63, batch=B)[:, 1:7].to(DEV)
    ctx = torch.cat([out, new], 1)
    L = ctx.shape[1]
    out2 = m.generate_continue(new, max_new_tokens=8, seed=seed + 50, **kw)
    toks2 = out2[:, L:]
    _, o2 = O.greedy_generate(osd, SMALL, ctx, vf.bfloat16(), toks2.shape[1], forced=toks2)
    _check_e2e(toks2, o2, [seed + 50 + b for b in range(B)], [L] * B, f"{fmt} continue", e2e_tally)
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
        _check_e2e(t, o3, [1000 + i], [p.numel()], f"{fmt} request {i}", e2e_tally)


def test_most_end_to_end_steps_are_decided(e2e_tally):
    assert e2e_tally[1] > 0 and e2e_tally[0] >= 0.5 * e2e_tally[1], e2e_tally

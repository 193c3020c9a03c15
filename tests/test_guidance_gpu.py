"""Classifier-free guidance on the GPU (guidance.cu, vcl_llm_set_guidance, generate(guidance_scale=...)).

Bars:
- vcl_op_guidance against float64 on the same fp32 rows: |out - ref| <= (|g| + |g - 1| + 1) * (1e-5 + 2^-21 * (|x_c -
  m_c| + |x_u - m_u| + |log S_c| + |log S_u|)) + 2^-22 * |ref|. Each fp32 log-softmax value carries the rounding of
  x - m, of log S (S summed in about 40 sequential fp32 adds per thread, then a 10-level tree: relative error below
  1e-6, so an absolute error in log S below 1e-6, plus expf / logf at 2 ulps) and of the final subtraction; the
  combination adds one rounding each for the difference, the product and the sum. Non-finite results (a NaN row, a
  row of -inf, g * inf) match float64's class exactly; rows without a partner are copied bit for bit;
- the guided token inside the CUDA-graph loops equals vcl_op_guidance then the arg-max / vcl_op_sample_ex on the
  logits vcl_llm_decode_step returns for the two clips at the same positions, bit for bit, and the partner clip is
  fed the same token;
- end to end, greedy guided generate against the oracle's logits of both sequences combined by HF's fp32 formula,
  teacher-forced on the engine's tokens: the same token wherever the oracle's guided top-1 / top-2 margin exceeds
  (|g| + |g - 1|) * 2 * delta, delta = 4 bf16 ulps of the larger row maximum (the bf16 logits' error moves each
  log-softmax by at most 2 delta);
- guidance_scale=1.0 is the unguided call (same tokens, same launch count), and after a guided call every path equals
  a fresh engine's.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import vcl_native as vn  # noqa: E402
from oracle import vcl_oracle as O  # noqa: E402
from _util import to_dev  # noqa: E402
from test_padded_batch_gpu import video_feats  # noqa: E402
from test_nucleus_gpu import SMALL, _bits, _gen, _model_at  # noqa: E402

DEV = "cuda"


@pytest.fixture(autouse=True)
def _release_device_memory():
    """engines allocate outside torch's caching allocator: drop each test's engines and torch's cache after it"""
    yield
    import gc
    gc.collect()
    torch.cuda.empty_cache()


def _ref(x, partner, g):
    """float64 restatement of the combination on fp32 rows x [B, V]"""
    x64 = x.double()
    lsm = torch.log_softmax(x64, dim=-1)
    out = x64.clone()
    for b, u in enumerate(partner):
        if u >= 0:
            out[b] = g[b] * (lsm[b] - lsm[u]) + lsm[u]
    return out, lsm


def _rows(B, V, seed):
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, V, generator=gen) * (1 + 5 * torch.rand(B, 1, generator=gen))).bfloat16().float()
    return x


@torch.no_grad()
@pytest.mark.parametrize("V", [32003, 1000])
@pytest.mark.parametrize("B", [1, 2, 5, 8, 32])
def test_op_matches_fp64(V, B):
    rng = np.random.default_rng(B * 7 + V)
    x = _rows(B, V, B + V)
    h = B // 2
    partner = [h + b if b < h else -1 for b in range(B)]
    g = [float(rng.choice([0.0, 1.5, 3.0, -0.5, 1.0, 7.25])) for _ in range(B)]
    if B >= 8:   # special rows: -inf stretches, a NaN, all equal, a +inf
        x[0, : V // 3] = float("-inf")
        x[h + 1, 5] = float("nan")
        x[2] = 0.75
        x[h + 3, : V // 2] = float("-inf")
        x[h + 2] = 1.0
        x[3, 7] = float("inf")
    out = vn.op_guidance(x.to(DEV), partner, g).cpu()
    ref, lsm = _ref(x, partner, g)
    for b in range(B):
        if partner[b] < 0:
            assert torch.equal(out[b].view(torch.int32), x[b].view(torch.int32)), b
            continue
        r, o = ref[b], out[b].double()
        fin = torch.isfinite(r)
        # non-finite results: the same class (NaN, +inf, -inf) as float64's
        assert torch.equal(torch.isnan(o), torch.isnan(r)), b
        assert torch.equal(o[torch.isinf(r)], r[torch.isinf(r)]), b
        if not fin.any():
            continue
        u = partner[b]
        xc, xu = x[b].double(), x[u].double()
        mc, mu = xc.max(), xu.max()
        lsc = torch.logsumexp(xc - mc, 0) if torch.isfinite(mc) else torch.tensor(0.0)
        lsu = torch.logsumexp(xu - mu, 0) if torch.isfinite(mu) else torch.tensor(0.0)
        k = abs(g[b]) + abs(g[b] - 1) + 1
        bound = k * (1e-5 + 2 ** -21 * ((xc - mc).abs() + (xu - mu).abs() + lsc.abs() + lsu.abs())) + 2 ** -22 * r.abs()
        err = (o - r).abs()
        assert bool((err[fin] <= bound[fin]).all()), (b, float(err[fin].max()), float(bound[fin].min()))
    # deterministic
    again = vn.op_guidance(x.to(DEV), partner, g).cpu()
    assert torch.equal(out.view(torch.int32), again.view(torch.int32))


def test_op_rejections():
    x = torch.zeros(4, 100, device=DEV)
    for partner, g in (([1, 0, -1, -1], [2.0] * 4), ([0, -1, -1, -1], [2.0] * 4), ([2, 2, -1, -1], [2.0] * 4),
                       ([2, -1, -1, -1], [float("inf")] * 4), ([9, -1, -1, -1], [2.0] * 4)):
        with pytest.raises(vn.VclError, match="vcl_op_guidance"):
            vn.op_guidance(x, partner, g)


def _flat(max_batch=4, fmt="bf16", seed=21):
    m = _model_at(480, fmt=fmt, max_batch=max_batch)
    m.load_state_dict(to_dev(O.random_llm_state(SMALL, seed=seed)))
    return m


def _text(seed, n):
    return torch.cat([torch.tensor([1]), torch.randint(3, 32000, (n - 1,), generator=torch.Generator().manual_seed(seed))])


@torch.no_grad()
@pytest.mark.parametrize("mode", ["greedy", "seeded", "nucleus_penalty", "logprobs"])
def test_in_graph_token_equals_ops_on_step_logits(mode):
    """generate's guided tokens (CUDA-graph loops) against decode_step's raw logits of both clips, combined by
    vcl_op_guidance and picked by the arg-max / vcl_op_sample_ex"""
    g = 1.75
    m = _flat()
    ids = O.make_prompt_ids(SMALL, 356, seed=31, batch=1).to(DEV)
    vf = video_feats(1, 32)
    neg = _text(33, 40)[None].to(DEV)
    n = 12
    kw = dict(eos_token_id=None, guidance_scale=g, negative_prompt_ids=neg)
    T, k, p, r, seed = 0.0, 0, 1.0, 1.0, 0
    if mode == "seeded":
        kw.update(do_sample=True, temperature=0.8, top_k=40, seed=5)
        T, k, seed = 0.8, 40, 5
    elif mode == "nucleus_penalty":
        kw.update(do_sample=True, temperature=0.7, top_k=0, top_p=0.9, repetition_penalty=1.3, seed=9)
        T, p, r, seed = 0.7, 0.9, 1.3, 9
    elif mode == "logprobs":
        kw.update(logprobs=5)
    out = _gen(m, ids, vf, n, **kw)
    S = ids.shape[1]
    toks = out[0, S:].tolist()
    lps = m.last_logprobs
    # replay: the same prefill, then one decode_step per token with the guidance table on; the logits are raw
    eng = m._engine
    ids2, pads2, spans, f2, shift = m._guided_batch(ids, None, vf, neg, None, None, eng.NV)
    assert shift == 0
    eng.set_guidance([0, 1], [1, -1], [g, 1.0])
    try:
        _, logits, tok = eng.prefill(ids2, f2, spans, want_logits=True, n_pad=pads2)
        seen = list(ids[0].tolist())
        for i in range(n):
            comb = vn.op_guidance(logits, [1, -1], [g, 1.0])
            if mode in ("greedy", "logprobs"):
                want = int(comb[0].argmax())
                if mode == "logprobs":
                    t2, _, lp = vn.op_sample_ex(comb[:1].contiguous(), [0.0], [0], [0], [S + i], [1.0], [1.0],
                                                top_n=[5])
                    assert int(t2[0]) == want
                    assert float(lp[0, 0]) == float(lps[0]["token_logprobs"][i]), i
            else:
                sets = _bits([set(seen)], SMALL.vocab) if r != 1.0 else None
                want = int(vn.op_sample_ex(comb[:1].contiguous(), [T], [k], [seed], [S + i], [p], [r],
                                           token_sets=sets)[0])
            assert toks[i] == want, (mode, i)
            assert int(tok[1]) == int(tok[0]), (mode, i)   # the handoff to the partner clip
            if mode in ("greedy", "logprobs"):             # (the replay's sampling entries are greedy)
                assert int(tok[0]) == want, (mode, i)
            seen.append(want)
            if i + 1 < n:
                logits, tok = eng.decode_step(torch.tensor([want, want], dtype=torch.int32, device=DEV), S + i,
                                              want_logits=True)
    finally:
        eng.set_guidance([0, 1], [-1, -1], [1.0, 1.0])


def _oracle_check(osd, ids, vf, neg, nf, toks, g, what, tally):
    """teacher-forced: the engine's tokens against the oracle's guided arg-max at every decided step"""
    n = toks.shape[1]
    _, oc = O.greedy_generate(osd, SMALL, ids, vf, n, forced=toks)
    _, ou = O.greedy_generate(osd, SMALL, neg, nf, n, forced=toks)
    for i in range(n):
        c, u = oc[i][0].float(), ou[i][0].float()
        s = g * (torch.log_softmax(c, -1) - torch.log_softmax(u, -1)) + torch.log_softmax(u, -1)
        top = torch.topk(s, 2).values
        mx = max(float(c.abs().max()), float(u.abs().max()))
        delta = 4 * 2.0 ** (math.floor(math.log2(mx)) - 7)
        bound = (abs(g) + abs(g - 1)) * 2 * delta
        margin = float(top[0] - top[1])
        tally["margins"].append(margin)
        tally["all"] += 1
        if margin > bound:
            tally["decided"] += 1
            assert int(toks[0, i]) == int(s.argmax()), (what, i, margin, bound)


@pytest.fixture(scope="module")
def tally():
    t = dict(all=0, decided=0, margins=[])
    yield t
    m = np.array(t["margins"]) if t["margins"] else np.zeros(1)
    print(f"guided e2e: {t['decided']} of {t['all']} steps decided; margins median {np.median(m):.3f}, "
          f"min {m.min():.4f}, max {m.max():.3f}")


@torch.no_grad()
@pytest.mark.parametrize("fmt", ["bf16", "fp8_e4m3"])
@pytest.mark.parametrize("B", [1, 8])
def test_end_to_end_matches_oracle(fmt, B, tally):
    from test_sampling_gpu import peaked_state
    import _fp8_ref as F8
    sd = to_dev(peaked_state())
    osd = sd if fmt == "bf16" else F8.dequantize_state(sd)
    m = _model_at(480, fmt=fmt, max_batch=2 * B)
    m.load_state_dict(dict(sd))
    g, n = 1.5, 8
    ids = O.make_prompt_ids(SMALL, 356, seed=41 + B, batch=B).to(DEV)
    vf = video_feats(B, 42)
    S = ids.shape[1]
    text_neg = torch.stack([_text(50 + b, 30 + 3 * b) for b in range(B)]) if B == 1 else \
        torch.stack([_text(50 + b, 40) for b in range(B)])
    noised = (vf + 0.5 * video_feats(B, 43)).half().float()
    for kind in ("text", "default", "video"):
        if kind == "text":
            kw = dict(negative_prompt_ids=text_neg.to(DEV))
        elif kind == "default":
            kw = {}
        else:
            kw = dict(negative_prompt_ids=ids, negative_video_spatio_temporal_features=noised)
        out = _gen(m, ids, vf, n, eos_token_id=None, guidance_scale=g, **kw)
        assert out.shape == (B, S + n) and torch.equal(out[:, :S], ids)
        toks = out[:, S:]
        for b in range(B if B == 1 else 2):
            neg = (text_neg[b:b + 1].to(DEV) if kind == "text" else ids[b:b + 1, -1:] if kind == "default"
                   else ids[b:b + 1])
            nf = noised[b:b + 1].bfloat16() if kind == "video" else None
            _oracle_check(osd, ids[b:b + 1], vf[b:b + 1].bfloat16(), neg, nf, toks[b:b + 1], g,
                          f"{fmt} B={B} {kind} row {b}", tally)


@torch.no_grad()
def test_most_steps_decided(tally):
    assert tally["all"] > 0 and tally["decided"] >= 0.5 * tally["all"], (tally["decided"], tally["all"])


@torch.no_grad()
def test_scale_one_is_unguided_and_guided_leaves_a_fresh_engine():
    ids = O.make_prompt_ids(SMALL, 356, seed=5, batch=2).to(DEV)
    vf = video_feats(2, 6)
    neg = torch.stack([_text(60 + b, 20) for b in range(2)]).to(DEV)
    for kw in (dict(eos_token_id=None), dict(do_sample=True, temperature=0.7, top_k=50, seed=11, eos_token_id=None)):
        fresh = _flat()
        a = _gen(fresh, ids, vf, 16, **kw)
        n0 = vn.launch_count()
        a2 = _gen(fresh, ids, vf, 16, **kw)
        la = vn.launch_count() - n0
        n0 = vn.launch_count()
        one = _gen(fresh, ids, vf, 16, guidance_scale=1.0, negative_prompt_ids=neg, **kw)
        l1 = vn.launch_count() - n0
        assert torch.equal(a, a2) and torch.equal(a, one) and la == l1
        used = _flat()
        _gen(used, ids, vf, 16, guidance_scale=2.5, negative_prompt_ids=neg, **kw)
        _gen(used, ids, vf, 16, **kw)            # the default graphs captured
        n0 = vn.launch_count()
        b = _gen(used, ids, vf, 16, **kw)
        lb = vn.launch_count() - n0
        assert torch.equal(a, b) and la == lb
        # the other paths: stopping criteria on the host, unseeded sampling, in flight
        crit = [lambda out, _s: out.shape[1] >= ids.shape[1] + 5]
        assert torch.equal(_gen(fresh, ids, vf, 16, stopping_criteria=crit, **kw),
                           _gen(used, ids, vf, 16, stopping_criteria=crit, **kw))
        reqs = [dict(input_ids=_text(70, 30), max_new_tokens=6), dict(input_ids=_text(71, 25), max_new_tokens=9)]
        ra = fresh.generate_requests(reqs, eos_token_id=None)
        rb = used.generate_requests(reqs, eos_token_id=None)
        assert all(torch.equal(x.cpu(), y.cpu()) for x, y in zip(ra, rb))


@torch.no_grad()
def test_guided_paths_and_continuation():
    """stopping criteria (host chunking), unseeded sampling (host guidance) and a longer negative prompt run; the
    continuation of a guided call is the unguided continuation of the same conversation"""
    m = _flat(max_batch=4)
    ids = O.make_prompt_ids(SMALL, 356, seed=7, batch=2).to(DEV)
    vf = video_feats(2, 8)
    S = ids.shape[1]
    neg = torch.stack([_text(80 + b, 20) for b in range(2)]).to(DEV)
    full = _gen(m, ids, vf, 20, eos_token_id=None, guidance_scale=2.0, negative_prompt_ids=neg)
    crit = [lambda out, _s: out.shape[1] >= S + 7]
    cut = _gen(m, ids, vf, 20, eos_token_id=None, guidance_scale=2.0, negative_prompt_ids=neg, stopping_criteria=crit)
    assert torch.equal(cut, full[:, :S + 7])
    # the host path: HF's formula on the step logits, the negative clips fed the same tokens
    torch.manual_seed(3)
    smp = _gen(m, ids, vf, 10, eos_token_id=None, guidance_scale=2.0, negative_prompt_ids=neg, do_sample=True,
               temperature=1e-4, top_k=1)
    assert torch.equal(smp, full[:, :S + 10])
    # a negative prompt longer than the prompt: the prompts are padded on the left, the result is not
    long_neg = torch.stack([_text(90 + b, S + 10) for b in range(2)]).to(DEV)
    lo = _gen(m, ids, vf, 6, eos_token_id=None, guidance_scale=2.0, negative_prompt_ids=long_neg)
    assert lo.shape == (2, S + 6) and torch.equal(lo[:, :S], ids)
    # continuation: generate_continue after the guided call continues the prompts' rows without guidance, as after
    # an unguided call: teacher-forced against the oracle on the whole conversation, the same token at every step
    # whose top-2 margin exceeds 4 bf16 ulps
    _gen(m, ids, vf, 12, eos_token_id=None, guidance_scale=2.0, negative_prompt_ids=neg)
    new = _text(99, 6)[None].expand(2, 6).to(DEV)
    c1 = m.generate_continue(new, max_new_tokens=8, eos_token_id=None)
    L = S + 12 + 6
    assert c1.shape == (2, L + 8) and torch.equal(c1[:, :S + 12], full[:, :S + 12])
    osd = to_dev(O.random_llm_state(SMALL, seed=21))
    decided = 0
    for b in range(2):
        _, lg = O.greedy_generate(osd, SMALL, c1[b:b + 1, :L], vf[b:b + 1].bfloat16(), 8, forced=c1[b:b + 1, L:])
        for i in range(8):
            x = lg[i][0].float()
            top = torch.topk(x, 2).values
            if float(top[0] - top[1]) > 4 * 2.0 ** (math.floor(math.log2(float(top[0].abs()) + 1e-30)) - 7):
                decided += 1
                assert int(c1[b, L + i]) == int(x.argmax()), (b, i)
    assert decided >= 4


def test_rejections_before_device_work():
    m = _flat(max_batch=2)
    ids = O.make_prompt_ids(SMALL, 0, seed=1, batch=2).to(DEV)
    with pytest.raises(ValueError, match="max_batch"):
        m.generate(ids, guidance_scale=2.0, max_new_tokens=2)
    with pytest.raises(ValueError, match="guidance_scale"):
        m.generate(ids[:1], guidance_scale=float("nan"), max_new_tokens=2)
    with pytest.raises(NotImplementedError, match="num_beams"):
        m.generate(ids[:1], guidance_scale=2.0, num_beams=2, max_new_tokens=2)
    eng = m._ensure_engine(need_llm=True)
    for clips, partner in (([0, 1], [1, 0]), ([0], [0]), ([0], [5])):
        with pytest.raises(vn.VclError, match="vcl_llm_set_guidance"):
            eng.set_guidance(clips, partner, [2.0] * len(clips))
    with pytest.raises(vn.VclError, match="not finite"):
        eng.set_guidance([0], [1], [float("inf")])

"""Classifier-free guidance on the host: the torch restatement (_guidance_ref) against transformers' processor, the
argument checks of generate, the negative prompt video_chatgpt_infer builds, and the stepwise path's host guidance
against the reference chain (guidance, then HF's processors)."""
import pytest
import torch

import _guidance_ref as GR
import _bans_ref as BR
from test_nucleus_cpu import _fake_model, _hf

V = 32003


class _Uncond:
    """a model for HF's processor: returns scripted logits and records what it was called with"""

    def __init__(self, rows):
        self.rows, self.calls = rows, []

    def __call__(self, input_ids, attention_mask=None, use_cache=True, past_key_values=None):
        self.calls.append((input_ids.clone(), attention_mask.clone()))
        lg = self.rows[len(self.calls) - 1][:, None, :].expand(-1, input_ids.shape[1], -1)
        return {"logits": lg, "past_key_values": len(self.calls)}


class _Out(dict):
    def __getattr__(self, k):
        return self[k]


@pytest.mark.parametrize("g", [0.0, 1.5, 3.0, -0.7, 7.25])
@pytest.mark.parametrize("neg", [False, True])
def test_restatement_matches_transformers(g, neg):
    transformers = pytest.importorskip("transformers")
    from transformers.generation.logits_process import UnbatchedClassifierFreeGuidanceLogitsProcessor as U
    gen = torch.Generator().manual_seed(int(g * 100) + neg)
    B, steps = 3, 4
    cond = [torch.randn(B, V, generator=gen) * 4 for _ in range(steps)]
    unc = [torch.randn(B, V, generator=gen) * 4 for _ in range(steps)]
    unc[1][0, :100] = float("-inf")
    fake = _Uncond(unc)
    model = lambda *a, **k: _Out(fake(*a, **k))   # noqa: E731
    ids = torch.randint(3, 32000, (B, 20), generator=gen)
    nids = torch.randint(3, 32000, (B, 7), generator=gen) if neg else None
    proc = U(g, model, nids, None)
    for t in range(steps):
        got = proc(ids, cond[t].clone())
        want = GR.guide(cond[t], unc[t], g)
        torch.testing.assert_close(got, want, rtol=0, atol=0, equal_nan=True, msg=f"step {t}")
        ids = torch.cat([ids, got.argmax(-1, keepdim=True)], 1)
    # the unconditional context: the negative prompt, or each row's last prompt token alone; then one token a step
    first = fake.calls[0][0]
    assert torch.equal(first, nids if neg else GR.default_negative(ids[:, :20]))
    assert all(c[0].shape[1] == 1 for c in fake.calls[1:])


@pytest.mark.parametrize("kw,exc,msg", [
    (dict(guidance_scale=float("nan")), ValueError, "guidance_scale"),
    (dict(guidance_scale=float("inf")), ValueError, "guidance_scale"),
    (dict(guidance_scale=2.0, num_beams=2), NotImplementedError, "num_beams"),
    (dict(guidance_scale=2.0, negative_prompt_ids=torch.ones(3, 4, dtype=torch.long)), ValueError,
     "negative_prompt_ids"),
    (dict(guidance_scale=2.0, negative_prompt_ids=torch.ones(2, 4, dtype=torch.long),
          negative_prompt_attention_mask=torch.ones(2, 5, dtype=torch.long)), ValueError, "attention_mask"),
    (dict(guidance_scale=2.0, negative_prompt_attention_mask=torch.ones(2, 5, dtype=torch.long)), ValueError,
     "needs negative_prompt_ids"),
    (dict(guidance_scale=2.0, negative_prompt_ids=torch.ones(2, 4, dtype=torch.long),
          negative_video_spatio_temporal_features=torch.zeros(3, 356, 1024)), ValueError, "negative_video"),
    (dict(guidance_scale=2.0, negative_video_spatio_temporal_features=torch.zeros(2, 356, 1024)), ValueError,
     "negative_video"),
])
def test_rejections_before_any_device_call(kw, exc, msg):
    m, eng = _fake_model(slots=4)
    m._kv_blocks = 0
    ids = torch.randint(3, 100, (2, 10))
    with pytest.raises(exc, match=msg):
        m.generate(ids, max_new_tokens=4, **kw)
    assert eng.calls == []


def test_batch_and_vocabulary_limits():
    m, eng = _fake_model(slots=4)
    m._kv_blocks = 0
    with pytest.raises(ValueError, match="max_batch"):
        m.generate(torch.randint(3, 100, (3, 10)), max_new_tokens=4, guidance_scale=2.0)
    m.config.vocab_size = 60000
    with pytest.raises(ValueError, match="vocabulary"):
        m.generate(torch.randint(3, 100, (1, 10)), max_new_tokens=4, guidance_scale=2.0)
    assert eng.calls == []
    # off: None and 1.0 (HF adds no processor at 1)
    assert m._guidance_args(None, None, None, None, torch.zeros(3, 2), 4) is None
    assert m._guidance_args(1.0, None, None, None, torch.zeros(3, 2), 4) is None


def test_guided_batch_pads_and_spans():
    m, _ = _fake_model(slots=4)
    ids = torch.randint(3, 100, (2, 6))
    neg = torch.randint(3, 100, (2, 9))
    mask = torch.ones(2, 9, dtype=torch.long)
    mask[1, :4] = 0
    ids2, pads2, spans, f2, shift = m._guided_batch(ids, [0, 2], None, neg, mask, None, 356)
    assert shift == 3 and ids2.shape == (4, 9) and f2 is None
    assert torch.equal(ids2[:2, 3:], ids) and (ids2[:2, :3] == ids[:, :1]).all() and torch.equal(ids2[2:], neg)
    assert pads2 == [3, 5, 0, 4]
    assert spans.tolist() == [-1] * 4 or all(s < 0 for s in spans.tolist())
    # the default negative: the last prompt token, alone after its padding
    ids2, pads2, _, _, shift = m._guided_batch(ids, None, None, None, None, None, 356)
    assert shift == 0 and pads2 == [0, 0, 5, 5] and torch.equal(ids2[2:, -1], ids[:, -1])


def test_negative_prompt_of_video_chatgpt_infer():
    from video_chatgpt.constants import DEFAULT_VID_END_TOKEN, DEFAULT_VID_START_TOKEN, DEFAULT_VIDEO_PATCH_TOKEN
    from video_chatgpt.inference import build_prompt
    for se in (True, False):
        for tr in (None, "some words"):
            pos, _ = build_prompt("What happens?", "video-chatgpt_v1", 4, se, tr)
            neg, _ = build_prompt("What happens?", "video-chatgpt_v1", 4, se, tr, with_video=False)
            assert DEFAULT_VIDEO_PATCH_TOKEN * 4 in pos
            for t in (DEFAULT_VIDEO_PATCH_TOKEN, DEFAULT_VID_START_TOKEN, DEFAULT_VID_END_TOKEN):
                assert t not in neg
            span = (DEFAULT_VID_START_TOKEN if se else "") + DEFAULT_VIDEO_PATCH_TOKEN * 4 + \
                (DEFAULT_VID_END_TOKEN if se else "")
            assert neg == pos.replace("\n" + span, "")
            if tr:
                assert tr in neg


class _StepEngine:
    """decode_step over 2B rows with scripted logits; records the tokens fed"""

    def __init__(self, rows):
        self.rows, self.fed = rows, []

    def decode_step(self, tok, pos, want_logits=False):
        self.fed.append((tok.clone(), pos))
        return self.rows[len(self.fed)].clone(), tok


@pytest.mark.parametrize("sampled", [False, True])
def test_stepwise_host_guidance_matches_reference_chain(sampled):
    m, _ = _fake_model(slots=4)
    B, n, g, S = 2, 5, 2.5, 8
    gen = torch.Generator().manual_seed(5 + sampled)
    rows = [(torch.randn(2 * B, V, generator=gen) * 3).bfloat16().float() for _ in range(n + 1)]
    ids = torch.randint(3, 50, (B, S), generator=gen)
    bans = m._ban_args(2, [[7]], None, None)
    T, k, p, r = 0.7, 50, 0.9, 1.2
    eng = _StepEngine(rows)
    m._pos = S
    torch.manual_seed(11)
    out = m._stepwise(eng, ids, rows[0], n, sampled, T, None, None, None, k, p, r, bans, guidance=g)
    # the reference chain: guidance, then the penalty, the bans, temperature, top-k, top-p (HF's order)
    torch.manual_seed(11)
    ctx = ids.clone()
    for t in range(n):
        x = GR.guide(rows[t][:B], rows[t][B:], g)
        _, lg = _hf(ctx, x.clone(), T, k, p, r) if sampled else (None, None)
        if sampled:
            for b in range(B):
                for tok in BR.banned(ctx[b].tolist(), 2, [[7]]):
                    lg[b, tok] = float("-inf")
        else:
            from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor
            lg = RepetitionPenaltyLogitsProcessor(penalty=r)(ctx, x.clone())
            for b in range(B):
                for tok in BR.banned(ctx[b].tolist(), 2, [[7]]):
                    lg[b, tok] = float("-inf")
        nxt = torch.multinomial(torch.softmax(lg, -1), 1)[:, 0] if sampled else lg.argmax(-1)
        ctx = torch.cat([ctx, nxt[:, None]], 1)
        if not sampled:
            assert torch.equal(out[:, S + t], nxt), t
    # the negative clips are fed each row's token, at the same cache column
    for t, (tok, pos) in enumerate(eng.fed):
        assert torch.equal(tok[:B], tok[B:]) and torch.equal(tok[:B].long(), out[:, S + t]) and pos == S + t

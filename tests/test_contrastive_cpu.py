"""CPU tests of contrastive search: the float64 rule (_contrastive_ref.py) on hand-built cases, the oracle-driven
restatement on a tiny oracle model (it must pick differently from greedy somewhere), and generate()'s argument
checks, each raised before any device work."""
import os

import numpy as np
import pytest
import torch

import _contrastive_ref as CR
from oracle import vcl_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V = 64


def test_candidates_ties_go_to_the_lower_id():
    z = np.array([0.0, 2.0, 1.0, 2.0, np.nan, 1.0, -np.inf])
    tok, p = CR.candidates(z, 4)
    assert tok.tolist() == [1, 3, 2, 5]
    assert p[0] == p[1] and p[2] == p[3]
    assert abs(CR.probs(z)[~np.isnan(z)].sum() - 1.0) < 1e-12 and CR.probs(z)[4] == 0.0


def test_rank_ties_between_candidates_go_to_the_lower_j():
    ctx = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    g = np.array([[0.0, 0.0, 1.0], [0.0, 0.0, 2.0], [1.0, 1.0, 0.0]])
    s, score, j = CR.rank(ctx, g, [0.3, 0.3, 0.3], 0.5)
    assert s.tolist() == [0.0, 0.0, pytest.approx(2 ** -0.5)]
    assert score[0] == score[1] and j == 0


def test_pad_rows_are_not_context():
    """a row parallel to candidate 0 in the padding would make it lose; without it candidate 0 wins"""
    real = np.array([[1.0, 0.0, 0.0]])
    pad = np.array([[0.0, 0.0, 1.0]])
    g = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0]])
    p = [0.5, 0.4]
    assert CR.rank(real, g, p, 0.6)[2] == 0
    assert CR.rank(np.concatenate([pad, real]), g, p, 0.6)[2] == 1


def test_alpha_one_is_the_pure_degeneration_penalty():
    rng = np.random.default_rng(3)
    ctx, g = rng.standard_normal((20, 16)), rng.standard_normal((6, 16))
    p = rng.random(6)
    s, score, j = CR.rank(ctx, g, p, 1.0)
    assert j == int(np.argmin(s)) and np.allclose(score, -s)


def test_alpha_near_zero_is_greedy():
    rng = np.random.default_rng(4)
    for _ in range(20):
        z = rng.standard_normal(V) * 3
        tok, p = CR.candidates(z, 5)
        s, score, j = CR.rank(rng.standard_normal((9, 8)), rng.standard_normal((5, 8)), p, 1e-9)
        assert tok[j] == int(np.argmax(z))


def test_oracle_restatement_differs_from_greedy():
    """on a tiny random oracle model, contrastive search (teacher forced with its own picks) follows greedy at alpha ~ 0 and picks
    a non-greedy candidate at some step for alpha 0.6"""
    cfg = O.LlmCfg(hidden=64, inter=128, heads=2, layers=2, vocab=V)
    sd = O.random_llm_state(cfg, seed=7)
    differs = 0
    for seed in range(3):
        ids = torch.randint(3, V, (1, 12), generator=torch.Generator().manual_seed(seed))
        step, ctx0, z0 = CR.oracle_step_fn(sd, cfg, ids, None)
        greedy, _ = O.greedy_generate(sd, cfg, ids, None, 8)
        near0 = CR.generate(step, ctx0, z0, 4, 1e-9, 8)
        assert [st["token"] for st in near0] == greedy[0].tolist()
        out = CR.generate(step, ctx0, z0, 4, 0.6, 8)
        differs += sum(st["pick"] != 0 for st in out)
    assert differs > 0


class NoDevice:
    NV = 356

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *a, **k: self.calls.append(name)


def _model(eng, max_batch=16, vocab=V):
    from video_chatgpt.model import VideoChatGPTConfig, VideoChatGPTLlamaForCausalLM
    cfg = VideoChatGPTConfig(hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                             vocab_size=vocab)
    m = VideoChatGPTLlamaForCausalLM(cfg, clip_config={}, max_batch=max_batch, max_seq=128)
    vc = m.get_model().vision_config
    vc.vid_patch_token, vc.vid_start_token, vc.vid_end_token, vc.use_vid_start_end = vocab + 1, vocab + 2, vocab + 3, True
    m.device = torch.device("cpu")
    m._engine, m._llm_loaded = eng, True
    return m


@pytest.mark.parametrize("kw,exc,match", [
    (dict(penalty_alpha=0.6, do_sample=True), NotImplementedError, "do_sample"),
    (dict(penalty_alpha=0.6, seed=3), NotImplementedError, "seed"),
    (dict(penalty_alpha=0.6, num_beams=2), NotImplementedError, "num_beams"),
    (dict(penalty_alpha=0.6, guidance_scale=1.5), NotImplementedError, "guidance_scale"),
    (dict(penalty_alpha=0.6, logprobs=2), NotImplementedError, "logprobs"),
    (dict(penalty_alpha=0.6, top_p=0.9), NotImplementedError, "top_p"),
    (dict(penalty_alpha=0.6, repetition_penalty=1.2), NotImplementedError, "repetition_penalty"),
    (dict(penalty_alpha=0.6, no_repeat_ngram_size=2), NotImplementedError, "no_repeat_ngram_size"),
    (dict(penalty_alpha=0.6, bad_words_ids=[[5]]), NotImplementedError, "bad_words_ids"),
    (dict(penalty_alpha=0.6, min_new_tokens=2), NotImplementedError, "min_new_tokens"),
    (dict(penalty_alpha=0.6), ValueError, "max_batch"),                 # HF's top_k 50 > max_batch 16
    (dict(penalty_alpha=0.6, top_k=65), ValueError, "65"),
    (dict(penalty_alpha=1.5, top_k=4), ValueError, "penalty_alpha"),
    (dict(penalty_alpha=-0.1, top_k=4), ValueError, "penalty_alpha"),
    (dict(penalty_alpha="0.5", top_k=4), ValueError, "penalty_alpha"),
    (dict(penalty_alpha=0.6, top_k=4.0), ValueError, "top_k"),
    (dict(penalty_alpha=0.6, top_k=4, max_new_tokens=200, input_ids=torch.ones(1, 128, dtype=torch.int64)),
     ValueError, "max_seq"),
])
def test_rejections_before_any_device_work(kw, exc, match):
    eng = NoDevice()
    m = _model(eng)
    ids = kw.pop("input_ids", torch.tensor([[1, 5, 6]]))
    with pytest.raises(exc, match=match):
        m.generate(ids, **kw)
    assert eng.calls == []


def test_vocabulary_limit_is_checked_first():
    import vcl_native as vn
    eng = NoDevice()
    m = _model(eng, vocab=vn.SAMPLE_WIDE_MAX_V + 1)
    with pytest.raises(ValueError, match="vocabulary"):
        m.generate(torch.tensor([[1, 5, 6]]), penalty_alpha=0.6, top_k=4)
    assert eng.calls == []


class _Reached(Exception):
    pass


@pytest.mark.parametrize("kw", [dict(), dict(penalty_alpha=None), dict(penalty_alpha=0), dict(penalty_alpha=0.0),
                                dict(penalty_alpha=0.6, top_k=1), dict(penalty_alpha=0.6, top_k=0)])
def test_calls_without_contrastive_search_take_the_old_paths(kw):
    m = _model(NoDevice())

    def cs(*a, **k):
        raise AssertionError("the contrastive path was taken")

    def engine(*a, **k):
        raise _Reached()

    m._contrastive_generate, m._ensure_engine = cs, engine
    with pytest.raises(_Reached):
        m.generate(torch.tensor([[1, 5, 6]]), **kw)


def test_generate_continue_after_contrastive_raises():
    m = _model(NoDevice())
    m._after_contrastive, m._last_out = True, torch.ones(1, 4, dtype=torch.int64)
    with pytest.raises(ValueError, match="contrastive"):
        m.generate_continue(torch.tensor([[1, 2]]))


def test_inference_passes_penalty_alpha_and_top_k_without_sampling():
    import inspect
    from video_chatgpt import inference
    sig = inspect.signature(inference.video_chatgpt_infer)
    assert sig.parameters["penalty_alpha"].default is None and sig.parameters["top_k"].default is None
    src = inspect.getsource(inference.video_chatgpt_infer)
    assert "do_sample = False" in src and "**contrastive" in src


def test_new_symbols_are_exported():
    import vcl_native as vn
    for name in ("vcl_llm_contrastive_start", "vcl_llm_contrastive_decode", "vcl_op_contrastive_rank"):
        assert name in vn.EXPORTED_SYMBOLS
    with open(os.path.join(ROOT, "include", "vcl.h")) as f:
        h = f.read()
    for name in ("vcl_llm_contrastive_start", "vcl_llm_contrastive_decode", "vcl_op_contrastive_rank"):
        assert name + "(" in h
